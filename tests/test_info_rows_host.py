"""CPU: the host side of the device-formatted ``.info`` rows (graphed.EvalRun.info) -- the question prefixes and the
entity name table (evaluate.InfoTables) against json.dumps of the rows the evaluator writes, the header declarations
and bindings of gr_info_rows_size / gr_info_rows_write with every refusal before any CUDA call, and a host build of
the float64 formatter (csrc/float_repr.cuh) against Python's repr.  The GPU half is tests/test_info_rows_gpu.py."""
import ctypes
import json
import math
import os
import subprocess

import numpy as np
import pytest

from gnn_rag_b200 import _build, _lib, evaluate, synthetic as S

from test_device_split_host import NE, SplitLoader

PTR = 0x1000          # a non-null device pointer: never dereferenced, every call below is refused first
ENT = {"e%d" % i: i for i in range(NE)}


class _Model:
    num_iter = 3


def _evaluator(tmp_path, **args):
    a = dict(S.model_args("ReaRev"), checkpoint_dir=str(tmp_path), experiment_name="x", eps=0.95, **args)
    return evaluate.Evaluator(a, _Model(), ENT, {"r0": 0}, "cpu")


def _row(ev, L, q, metrics, case, cand):
    """The per-batch evaluator's row of question q (Evaluator.write_info + Evaluator._row) as text."""
    L.sample_ids = np.array([q])
    obj = ev.write_info(L, None, ev.model.num_iter)[0]
    p, r, f1, hit, em = metrics
    obj["answers"] = [ev._name(a) for a in L.answer_lists[q]]
    obj["precison"], obj["recall"], obj["f1"], obj["hit"] = p, r, f1, hit
    obj["em"] = int(em) if case == 3 else em
    obj["cand"] = [(ev._name(e), float(pr)) for e, pr in cand]
    return json.dumps(obj) + "\n"


def _from_tables(t, q, metrics, case, cand):
    """The same row as csrc/info_rows.cu assembles it from the tables."""
    prefix = t["prefix"][t["prefix_off"][q]:t["prefix_off"][q + 1]].tobytes().decode()
    name = lambda e: t["names"][t["name_off"][t["name_slot"][e]]:t["name_off"][t["name_slot"][e] + 1]].tobytes()  # noqa: E731
    keys = ("precison", "recall", "f1", "hit", "em")
    nums = [repr(float(v)) for v in metrics]
    if case == 3:
        nums[4] = "1" if metrics[4] else "0"
    body = ", ".join('"%s": %s' % (k, v) for k, v in zip(keys, nums))
    cands = ", ".join("[%s, %s]" % (name(e).decode(), repr(float(pr))) for e, pr in cand)
    return prefix + body + ', "cand": [' + cands + "]}\n"


def test_tables_rebuild_the_evaluator_rows(tmp_path):
    L = SplitLoader(seed=5, num_questions=9, max_local_entity=30)
    L.answer_lists[2] = []
    L.answer_lists[3] = [int(L.candidate_entities[3, 1])] * 2
    L.sample_ids = np.array([7, 1])
    ev = _evaluator(tmp_path)
    t = evaluate.InfoTables.host_arrays(ev, L, L.num_data)
    assert L.sample_ids.tolist() == [7, 1]                  # restored
    assert t["prefix_off"].shape == (L.num_data + 1,) and t["prefix_off"][0] == 0
    ents = sorted(set(L.candidate_entities.ravel().tolist()) - {NE})
    assert t["name_off"].shape == (len(ents) + 1,)
    assert [int(s) for s in t["name_slot"][ents]] == list(range(len(ents)))
    assert (t["name_slot"][[e for e in range(t["name_slot"].size) if e not in set(ents)]] == -1).all()
    rs = np.random.RandomState(0)
    for q in range(L.num_data):
        row = [int(e) for e in L.candidate_entities[q] if e != NE]
        cand = [(e, np.float32(rs.rand() ** 9)) for e in row]
        for case, metrics in ((3, (0.5, 1 / 3, 0.4, 1.0, 1.0)), (3, (0.0, 0.0, 0.0, 0.0, 0.0)),
                              (1, (0.0, 1.0, 0.0, 1.0, 1.0)), (2, (1.0, 0.0, 0.0, 0.0, 0.0))):
            assert _from_tables(t, q, metrics, case, cand) == _row(ev, L, q, metrics, case, cand)


def test_tables_use_entity2name_and_keep_python_escaping(tmp_path, monkeypatch):
    import pickle
    rs = np.random.RandomState(3)
    alphabet = ['"', "\\", "\n", "\t", "\x00", "\x1f", "\x7f", "é", "ü", "€", "中", "\U0001F600", "\U00010348", "a",
                " ", "/", "'"]
    names = {}
    while len(names) < NE:
        names["".join(rs.choice(alphabet, rs.randint(0, 8))) + str(len(names))] = len(names)
    monkeypatch.chdir(tmp_path)
    with open("ent2id.pickle", "wb") as f:
        pickle.dump(names, f)
    L = SplitLoader(seed=6, num_questions=5, max_local_entity=20)
    a = dict(S.model_args("ReaRev"), checkpoint_dir=str(tmp_path), experiment_name="x", eps=0.95, data_folder="sr-x")
    ev = evaluate.Evaluator(a, _Model(), {i: i for i in range(NE)}, {"r0": 0}, "cpu")
    t = evaluate.InfoTables.host_arrays(ev, L, L.num_data)
    listed = list(names)
    for e in set(L.candidate_entities.ravel().tolist()) - {NE}:
        s = t["name_slot"][e]
        got = t["names"][t["name_off"][s]:t["name_off"][s + 1]].tobytes()
        assert got == json.dumps(listed[e]).encode() and got.isascii()
    for q in range(L.num_data):
        cand = [(int(e), np.float32(0.25)) for e in L.candidate_entities[q] if e != NE]
        assert _from_tables(t, q, (1.0, 1.0, 1.0, 1.0, 1.0), 0, cand) == _row(ev, L, q, (1.0,) * 5, 0, cand)


# ---- the entry points ------------------------------------------------------------------------------------------------

def _types(name):
    P, I64 = ctypes.c_void_p, ctypes.c_int64
    if name == "gr_info_rows_size":
        return [P] * 6 + [I64, P, I64, P, P, I64, P, I64, P, I64, P, P, P]
    return [P] * 5 + [I64, P, I64, P, P, P, I64, P, I64, P, P, I64, P, P, P, I64, P]


@pytest.mark.parametrize("name", ["gr_info_rows_size", "gr_info_rows_write"])
def test_header_declaration_and_binding(name):
    assert _lib.SIGNATURES[name] == (ctypes.c_int, _types(name))
    assert getattr(_lib.load(), name).argtypes == _types(name)


def _size(**over):
    a = dict(metrics=PTR, cases=PTR, counts=PTR, cand_off=PTR, cand_total=PTR, eval_status=PTR, num_data=10, cand=PTR,
             capacity=100, order=PTR, prefix_off=PTR, num_q=10, name_slot=PTR, num_entity=50, name_off=PTR,
             num_names=40, row_off=PTR, summary=PTR, stream=None)
    a.update(over)
    lib = _lib.load()
    return lib.gr_info_rows_size(*a.values()), lib.gr_last_error().decode()


def _write(**over):
    a = dict(metrics=PTR, cases=PTR, counts=PTR, cand_off=PTR, cand_total=PTR, num_data=10, cand=PTR, capacity=100,
             order=PTR, prefix=PTR, prefix_off=PTR, num_q=10, name_slot=PTR, num_entity=50, names=PTR, name_off=PTR,
             num_names=40, row_off=PTR, summary=PTR, out=PTR, out_bytes=1000, stream=None)
    a.update(over)
    lib = _lib.load()
    return lib.gr_info_rows_write(*a.values()), lib.gr_last_error().decode()


_SIZES = "need num_data, capacity, num_q, num_entity and num_names >= 0"
_WSIZES = "need num_data, capacity, num_q, num_entity, num_names and out_bytes >= 0"


@pytest.mark.parametrize("over,msg", [
    *[(dict([(k, None)]), "null pointer") for k in ("metrics", "cases", "counts", "cand_off", "cand_total",
                                                     "eval_status", "cand", "order", "prefix_off", "name_slot",
                                                     "name_off")],
    (dict(row_off=None), "null output"), (dict(summary=None), "null output"),
    *[(dict([(k, -1)]), _SIZES) for k in ("num_data", "capacity", "num_q", "num_entity", "num_names")]])
def test_size_refusals(over, msg):
    assert _size(**over) == (-1, "gr_info_rows_size: invalid argument: " + msg)


@pytest.mark.parametrize("over,msg", [
    *[(dict([(k, None)]), "null pointer") for k in ("metrics", "cases", "counts", "cand_off", "cand_total", "cand",
                                                     "order", "prefix", "prefix_off", "name_slot", "names",
                                                     "name_off", "row_off", "summary")],
    (dict(out=None), "null output"),
    *[(dict([(k, -1)]), _WSIZES) for k in ("num_data", "capacity", "num_q", "num_entity", "num_names",
                                            "out_bytes")]])
def test_write_refusals(over, msg):
    assert _write(**over) == (-1, "gr_info_rows_write: invalid argument: " + msg)


# ---- the formatter on the host ---------------------------------------------------------------------------------------

def edge_values():
    """±0, the extreme subnormal and normal doubles, every power of ten and of two in range with both neighbours,
    both sides of the notation switches, a few repeating fractions, NaN and ±inf."""
    v = [0.0, 5e-324, 2.225073858507201e-308, 2.2250738585072014e-308, 1.7976931348623157e308, 0.3, 2 / 3, 1 / 3,
         0.1, 1.0, 1e-4, 1e-5, 1e16, 1e15, 9999999999999998.0, 123456789012345678.0, 7.300000288523734e-05,
         float("nan"), float("inf")]
    for e in range(-323, 309):
        p = float("1e%d" % e)
        v += [p, math.nextafter(p, 0.0), math.nextafter(p, math.inf)]
    for e in range(-1074, 1024):
        p = math.ldexp(1.0, e)
        v += [p, math.nextafter(p, 0.0), math.nextafter(p, math.inf)]
    for p in (1e-4, 1e-5, 1e16, 1e17):
        v += [math.nextafter(math.nextafter(p, 0.0), 0.0), math.nextafter(math.nextafter(p, math.inf), math.inf)]
    return v + [-x for x in v]


_HARNESS = r"""
#include "float_repr.cuh"
extern "C" void format_all(const double* x, long n, char* out, int* len) {
  for (long i = 0; i < n; ++i) {
    const gr::fr::Decimal d = gr::fr::shortest(x[i]);
    len[i] = gr::fr::repr_len(d);
    gr::fr::write_repr(d, out + i * gr::fr::kMaxReprLen);
  }
}
"""


def test_host_build_of_the_formatter_is_json_dumps(tmp_path):
    """The formatter's __host__ build (same source as the kernels'), compiled here by nvcc without a device."""
    src = tmp_path / "harness.cu"
    src.write_text(_HARNESS)
    _build.write_float_repr_table(str(tmp_path))
    so = str(tmp_path / "libharness.so")
    cmd = [_build._nvcc(), "-std=c++17", "-O2", "-Xcompiler", "-fPIC", "-shared", "-I", _build.CSRC, "-I",
           str(tmp_path), "-o", so, str(src)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    lib = ctypes.CDLL(so)
    rs = np.random.RandomState(0)
    x = np.array(edge_values() + rs.randint(0, 2 ** 62, 200000).view(np.float64).tolist()
                 + (rs.randint(1, 0x3F800001, 200000).astype(np.uint32).view(np.float32).astype(np.float64)).tolist())
    out = np.zeros(x.size * 24, dtype=np.uint8)
    n = np.zeros(x.size, dtype=np.int32)
    lib.format_all(x.ctypes.data_as(ctypes.c_void_p), ctypes.c_long(x.size), out.ctypes.data_as(ctypes.c_void_p),
                   n.ctypes.data_as(ctypes.c_void_p))
    buf = out.tobytes()
    got = [buf[24 * i:24 * i + n[i]].decode() for i in range(x.size)]
    want = [json.dumps(v) for v in x.tolist()]
    bad = [(v, g, w) for v, g, w in zip(x.tolist(), got, want) if g != w]
    assert not bad, bad[:10]
    assert {"NaN", "Infinity", "-Infinity", "-0.0", "5e-324", "1e-05", "0.0001", "1e+16",
            "9999999999999998.0"} <= set(got)
