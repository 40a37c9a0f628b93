"""The ``.info`` file of an evaluation epoch formatted on the device (graphed.EvalRun.info, csrc/info_rows.cu).

The formatter (csrc/float_repr.cuh) is held to ``repr`` / ``json.dumps`` through the row entry points on synthetic
records: float64 metrics and fp32 candidate probabilities over every fp32 binade below 1, random float64 bit patterns
and an edge list.  ``Evaluator(step=...)`` writes files byte-identical to the per-batch evaluator's for ReaRev, NSM
and GraftNet, int32 and int64 indices, batch sizes around the split, eps 1 and 1e-6, every case of f1_and_hits, after
an Adam step, and with escaped ``entity2name`` names; a shuffled split's rows equal the evaluator's rows of its
records.  A malformed run raises ``check()``'s message and writes no file, and the host tables are built once per
split."""
import json
import os
import pickle

import numpy as np
import pytest
import torch

from gnn_rag_b200 import evaluate, graphed, loader, ops, synthetic as S

from test_eval_epoch_gpu import _assert_same_as_per_batch, _evaluator, _loader, _model
from test_device_split_host import NE
from test_info_rows_host import edge_values

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")


# ---- the formatter through the row entry points ------------------------------------------------------------------

class _Tables:
    """One question whose prefix is "{" and one entity (0) named "a"."""

    def __init__(self):
        T = lambda a, dt: torch.tensor(a, dtype=dt, device=dev)       # noqa: E731
        self.prefix, self.prefix_off = T(list(b"{"), torch.uint8), T([0, 1], torch.int64)
        self.names, self.name_off = T(list(b'"a"'), torch.uint8), T([0, 3], torch.int64)
        self.name_slot = T([0], torch.int32)


def _format_rows(metrics, counts, probs):
    """Rows of synthetic records through gr_info_rows_size / gr_info_rows_write: ``metrics`` float64 [n, 5] (case 0,
    so em is a float), ``counts`` candidates per row, ``probs`` fp32 [sum(counts)] -> the bytes."""
    n = metrics.shape[0]
    i64 = dict(dtype=torch.int64, device=dev)
    counts = np.asarray(counts, dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    cand = torch.zeros(max(int(counts.sum()), 1), 2, **i64)
    if probs.size:
        bits = torch.from_numpy(probs.astype(np.float32).view(np.int32).astype(np.int64)).to(dev)
        cand[:probs.size, 1] = bits << 32
    recs = (torch.from_numpy(metrics).to(dev), torch.zeros(n, dtype=torch.int8, device=dev),
            torch.from_numpy(counts.astype(np.int32)).to(dev), torch.from_numpy(off).to(dev),
            torch.tensor([int(counts.sum())], **i64))
    order = torch.zeros(n, **i64)
    tables = _Tables()
    row_off, summary = torch.empty(n + 1, **i64), torch.empty(2, **i64)
    ops.info_rows_size(*recs, torch.zeros(4, dtype=torch.int32, device=dev), cand, order, tables, row_off, summary)
    total, flags = summary.tolist()
    assert flags == 0
    out = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
    ops.info_rows_write(*recs, cand, order, tables, row_off, summary, out)
    return out[:total].cpu().numpy().tobytes()


def _numbers(data):
    """The metric and candidate number strings of every row of _format_rows' output."""
    mets, cands = [], []
    for row in data.decode().splitlines():
        head, _, tail = row.partition(', "cand": [')
        mets += [p.partition(": ")[2] for p in head[1:].split(", ")]
        cands += [c.split("]")[0] for c in tail[:-2].split('["a", ')[1:]]
    return mets, cands


def _json_reprs(values):
    """json.dumps of every float64 of ``values``: repr, with NaN and the infinities as json.dumps writes them."""
    special = {"nan": "NaN", "inf": "Infinity", "-inf": "-Infinity"}
    return [special.get(r, r) for r in map(float.__repr__, values.tolist())]


def _check_values(metrics, counts, probs):
    data = _format_rows(metrics, counts, probs)
    mets, cands = _numbers(data)
    want_m, want_c = _json_reprs(metrics.ravel()), _json_reprs(probs.astype(np.float64))
    bad = [(w, g) for w, g in zip(want_m, mets) if w != g][:5] + [(w, g) for w, g in zip(want_c, cands) if w != g][:5]
    assert not bad
    assert len(mets) == len(want_m) and len(cands) == len(want_c)
    return data


def test_fp32_probabilities_over_every_binade():
    rs = np.random.RandomState(0)
    n = 1 << 24
    bits = rs.randint(1, 0x3F800001, n).astype(np.uint32)           # uniform over the patterns: every binade alike
    first = np.arange(0, 127, dtype=np.uint32) << 23                  # each binade's first and last pattern
    bits[:254] = np.concatenate([np.maximum(first, 1), first | 0x7FFFFF])
    bits[254] = 0x3F800000                                             # 1.0
    probs = bits.view(np.float32)
    rows = 4096
    counts = np.full(rows, n // rows)
    counts[0] -= 100
    counts[1] += 100
    counts[2] += counts[3]
    counts[3] = 0                                                      # a row without candidates
    metrics = rs.rand(rows, 5)
    _check_values(metrics, counts, probs)


def test_random_float64_bit_patterns_and_edges():
    rs = np.random.RandomState(1)
    n = 1 << 22
    vals = rs.randint(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64).view(np.float64)
    edge = np.array(edge_values())
    vals = np.concatenate([vals, edge, np.zeros((-(n + edge.size)) % 5)])
    metrics = vals.reshape(-1, 5)
    counts = np.zeros(metrics.shape[0], dtype=np.int64)
    counts[:3] = 1
    f32 = np.array([0.1, 7.3e-05, 1e-45], dtype=np.float32)
    data = _check_values(metrics, counts, f32)
    for s in (b"NaN", b"Infinity", b"-Infinity", b"-0.0", b"5e-324", b"1e-05", b"0.0001", b"1e+16",
              b"9999999999999998.0", b"0.10000000149011612", b"7.300000288523734e-05", b"1.401298464324817e-45"):
        assert s in data, s


# ---- whole files against the per-batch evaluator -----------------------------------------------------------------

@pytest.mark.parametrize("name,index_dtype,B,eps", [
    ("ReaRev", torch.int32, 1, 0.95), ("ReaRev", torch.int64, 7, 1.0), ("NSM", torch.int32, 64, 1e-6),
    ("NSM", torch.int64, 7, 0.95), ("GraftNet", torch.int32, 7, 1.0), ("GraftNet", torch.int64, 3, 1e-6)])
def test_files_equal_the_per_batch_evaluator(name, index_dtype, B, eps, tmp_path):
    L = _loader(name, num_questions=23, seed=5)
    m = _model(name, L)
    split = loader.DeviceSplit(L, dev, index_dtype=index_dtype)
    step = graphed.GraphedStep(m, NE, eps=eps)
    want = _assert_same_as_per_batch(name, m, L, split, B, eps, tmp_path, step)
    if eps >= 0.95:
        assert set(want[1]) == {0, 1, 2, 3}


def test_file_after_an_adam_step(tmp_path):
    L = _loader("NSM", num_questions=19)
    m = _model("NSM", L)
    split = loader.DeviceSplit(L, dev)
    step = graphed.GraphedStep(m, NE, eps=0.95)
    first = _assert_same_as_per_batch("NSM", m, L, split, 5, 0.95, tmp_path, step)
    params = [p for p in m.parameters() if p.requires_grad]
    g = torch.Generator(device=dev).manual_seed(4)
    for p in params:
        p.grad = torch.randn(p.shape, device=dev, generator=g)
    torch.optim.Adam(params, lr=2e-2).step()
    second = _assert_same_as_per_batch("NSM", m, L, split, 5, 0.95, tmp_path, step)
    assert second[2] != first[2]


def test_shuffled_split_rows_are_the_rows_of_its_records(tmp_path):
    """The fact order of a shuffled split comes from seeds drawn in the graphs, so the per-batch evaluator does not
    replay it: the device rows are held to the evaluator's rows (write_info + _row) of the run's own records."""
    L = _loader("GraftNet")
    m = _model("GraftNet", L)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    step = graphed.GraphedStep(m, NE, eps=0.95)
    ev = _evaluator("GraftNet", m, L, tmp_path, "shuffled", 0.95, step=step)
    torch.manual_seed(9)
    run = step.start_eval(split, 4)
    prec, rec, f1, hit, em, cases, retrieved = run.result()
    path = str(tmp_path / "want.info")
    ev.file_write = open(path, "w")
    for start in range(0, L.num_data, 4):
        L.sample_ids = L.batches[start:min(start + 4, L.num_data)]
        objs = ev.write_info(split, None, m.num_iter)
        for b, answers in enumerate(L.answer_lists[L.sample_ids]):
            i = start + b
            e = int(em[i]) if cases[i] == 3 else float(em[i])
            ev._row(objs[b], list(answers), float(prec[i]), float(rec[i]), float(f1[i]), float(hit[i]), e,
                    retrieved[i])
    ev.file_write.close()
    got = tmp_path / "got.info"
    with open(str(got), "wb") as f:
        assert run.info(ev.info_tables(split), f) is None
    assert got.read_bytes() == open(path, "rb").read()
    assert run.info(ev.info_tables(split)).tobytes() == got.read_bytes()


def test_entity2name_with_escapes(tmp_path, monkeypatch):
    rs = np.random.RandomState(2)
    alphabet = ['"', "\\", "\n", "\r", "\x00", "\x1b", "é", "ß", "€", "中", "�", "\U0001F600", "\U00010348", "a",
                "/", " "]
    names = {}
    while len(names) < NE:
        names["".join(rs.choice(alphabet, rs.randint(0, 10))) + "#%d" % len(names)] = len(names)
    monkeypatch.chdir(tmp_path)
    with open("ent2id.pickle", "wb") as f:
        pickle.dump(names, f)
    L = _loader("ReaRev")
    m = _model("ReaRev", L)
    split = loader.DeviceSplit(L, dev)
    step = graphed.GraphedStep(m, NE, eps=1.0)
    files = []
    for tag, st in (("batch", None), ("epoch", step)):
        args = dict(S.model_args("ReaRev"), checkpoint_dir=str(tmp_path), experiment_name=tag, eps=1.0,
                    data_folder="sr-test")
        ev = evaluate.Evaluator(args, m, {i: i for i in range(NE)}, {"r%d" % i: i for i in range(L.num_kb_relation)},
                                dev, step=st)
        out = ev.evaluate(split, test_batch_size=4)
        files.append((out, ev.case_ct, open(os.path.join(str(tmp_path), tag + "_test.info"), "rb").read()))
    assert files[0] == files[1]
    assert b"\\u" in files[1][2] and b'\\"' in files[1][2] and b"\\\\" in files[1][2]


# ---- bad runs and the host tables --------------------------------------------------------------------------------

def test_bad_run_raises_and_writes_no_file(tmp_path):
    L = _loader("ReaRev")
    m = _model("ReaRev", L)
    split = loader.DeviceSplit(L, dev)
    step = graphed.GraphedStep(m, NE, eps=0.95)
    ev = _evaluator("ReaRev", m, L, tmp_path, "bad", 0.95, step=step)

    def bad_order(is_sequential=True):
        L.batches = np.arange(L.num_data)
        L.batches[5] = L.num_data + 7
    L.reset_batches = bad_order
    with pytest.raises(RuntimeError, match=r"DeviceSplit: batch assembly status 1 \(1: question id out of range"):
        ev.evaluate(split, test_batch_size=4)
    assert not os.path.exists(os.path.join(str(tmp_path), "bad_test.info"))
    run = step.start_eval(split, 4)
    with pytest.raises(RuntimeError, match="batch assembly status 1"):
        run.info(ev.info_tables(split))


def test_tables_are_built_once_per_split(tmp_path):
    L = _loader("ReaRev")
    m = _model("ReaRev", L)
    split = loader.DeviceSplit(L, dev)
    step = graphed.GraphedStep(m, NE, eps=0.95)
    ev = _evaluator("ReaRev", m, L, tmp_path, "twice", 0.95, step=step)
    calls = []
    get_quest = L.get_quest
    L.get_quest = lambda training=False: calls.append(1) or get_quest(training)
    first = ev.evaluate(split, test_batch_size=4)
    tables = ev.info_tables(split)
    data = open(os.path.join(str(tmp_path), "twice_test.info"), "rb").read()
    assert ev.evaluate(split, test_batch_size=4) == first
    assert open(os.path.join(str(tmp_path), "twice_test.info"), "rb").read() == data
    ev.evaluate(split, test_batch_size=5)
    assert len(calls) == 1 and ev.info_tables(split) is tables
    assert list(L.sample_ids) == list(L.batches[(L.num_data - 1) // 5 * 5:L.num_data])
