"""ctypes binding of libgnnrag_b200.so (include/gnnrag_b200.h).  No CPU fallback: if the library is
missing the import fails loudly."""
import ctypes
import os
import re

from . import _build

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "gnnrag_b200.h")

# C parameter / return type -> ctypes type; `const char*` binds as c_char_p and every other pointer as c_void_p
_CTYPES = {
    "int": ctypes.c_int,
    "int64_t": ctypes.c_int64,
    "uint32_t": ctypes.c_uint32,
    "size_t": ctypes.c_size_t,
    "double": ctypes.c_double,
}


def _ctype(decl, where):
    """ctypes type of a declaration such as `const float* table` or `int64_t` (`where` names it in errors)."""
    if "*" in decl:
        base, _, rest = decl.partition("*")
        if " ".join(base.split()) == "const char" and "*" not in rest:
            return ctypes.c_char_p
        return ctypes.c_void_p
    words = decl.split()
    for typ in (" ".join(words), " ".join(words[:-1])):   # without and with a parameter name
        if typ in _CTYPES:
            return _CTYPES[typ]
    raise ImportError("%s: no ctypes binding for type %r" % (where, " ".join(words)))


def parse_signatures(text):
    """name -> (restype, argtypes) for every `ret gr_name(params);` prototype of a C header."""
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"//[^\n]*", "", text)
    sigs = {}
    for m in re.finditer(r"((?:const\s+)?[A-Za-z_]\w*[\s*]+)\b(gr_\w+)\s*\(([^;{}()]*)\)\s*;", text):
        ret, name, params = m.group(1), m.group(2), m.group(3).strip()
        params = [] if params in ("", "void") else [p.strip() for p in params.split(",")]
        sigs[name] = (_ctype(ret, "%s: return type" % name),
                      [_ctype(p, "%s: parameter %d (%s)" % (name, i, p)) for i, p in enumerate(params)])
    return sigs


# name -> (restype, argtypes) of every entry point, read from include/gnnrag_b200.h
with open(HEADER) as _f:
    SIGNATURES = parse_signatures(_f.read())

_lib = None


def lib_path():
    return _build.LIB_PATH


def load(build_if_missing=True):
    """Load (building first if needed and possible).  Raises ImportError when unavailable."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if build_if_missing and _build.needs_build():
        try:
            _build.build()
        except Exception as e:  # noqa: BLE001
            if not os.path.exists(path):
                raise ImportError("libgnnrag_b200.so is not built and nvcc failed: %s" % e)
    if not os.path.exists(path):
        raise ImportError("libgnnrag_b200.so not found at %s (run `python -m gnn_rag_b200._build`)" % path)
    lib = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            raise ImportError("libgnnrag_b200.so does not export %s (stale build?)" % name)
        fn.restype = res
        fn.argtypes = args
    if lib.gr_abi_version() != 1:
        raise ImportError("libgnnrag_b200.so ABI version mismatch")
    _lib = lib
    return lib


class GrError(RuntimeError):
    pass


def check(rc):
    if rc != 0:
        msg = load().gr_last_error()
        raise GrError("libgnnrag_b200 error %d: %s" % (rc, msg.decode() if msg else "?"))
