"""CPU: the ctypes bindings are read from include/gnnrag_b200.h, so each argument binds with its C type."""
import ctypes
import re

import pytest

from gnn_rag_b200 import _build, _lib

I32, I64, U32, SZ, DBL, P = (ctypes.c_int, ctypes.c_int64, ctypes.c_uint32, ctypes.c_size_t, ctypes.c_double,
                             ctypes.c_void_p)


def test_pinned_prototypes_bind_to_their_c_types():
    sig = _lib.SIGNATURES
    assert sig["gr_csr_build"] == (I32, [P, P, P, I32, I64, I64, I64] + [P] * 11 + [SZ, P])
    assert sig["gr_graft_aggregate_backward_det_ex"] == (
        I32, [P] * 7 + [I64, P, I64, P, DBL, P, I64, P, P, I64, P, I64, I32, I32, I32] + [P] * 5
        + [I64, I64, P, SZ, U32, P])
    assert sig["gr_set_option"] == (I32, [ctypes.c_char_p, I64])
    assert sig["gr_last_error"] == (ctypes.c_char_p, [])
    assert sig["gr_lstm_max_hidden"] == (SZ, [])


def test_parser_reads_prototypes_and_skips_bodies_and_comments():
    text = """
    /* int gr_commented(int x); */
    static inline int64_t gr_pad4(int64_t n) { return (n + 3) & ~(int64_t)3; }
    size_t gr_a(void);
    int gr_b(const float* x, unsigned long long* y, int64_t n,   // a line comment
             double p, uint32_t flags, const char* name);
    """
    assert _lib.parse_signatures(text) == {
        "gr_a": (SZ, []),
        "gr_b": (I32, [P, P, I64, DBL, U32, ctypes.c_char_p]),
    }


@pytest.mark.parametrize("proto,where", [
    ("int gr_bad(int a, float b);", "gr_bad: parameter 1 (float b)"),
    ("float gr_bad(int a);", "gr_bad: return type"),
    ("int gr_bad(unsigned n);", "gr_bad: parameter 0 (unsigned n)"),
])
def test_unknown_type_raises_import_error(proto, where):
    with pytest.raises(ImportError, match="^" + re.escape(where)):
        _lib.parse_signatures(proto)


def test_every_prototype_in_the_header_binds():
    lib = ctypes.CDLL(_build.LIB_PATH)
    assert len(_lib.SIGNATURES) >= 70
    for name, (res, args) in _lib.SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
