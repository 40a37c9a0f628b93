"""Exact restatements of the rule-path kernels (csrc/rule_paths.cu), independent of every kernel and of the package:
gr_rule_adj_build's label-grouped adjacency, built straight from the triple list rather than from the CSR, and the
level expansion of gr_rule_level_count / gr_rule_level_emit / gr_rule_paths_write as ops.rule_walks drives it.

Everything here is integer work in numpy on the CPU.  tests/test_rule_paths_edges_gpu.py holds the kernels to these
bit for bit; tests/test_rule_paths_edges_host.py pins them to the networkx restatement of the reference
(tests/rule_paths_ref.py)."""
import numpy as np

_LAB = np.int64(2 ** 31)           # key = row * 2^31 + label: rows and labels are int32


# ---- gr_rule_adj_build -------------------------------------------------------------------------------------------------

def adjacency(heads, labs, tails, B, N):
    """The label-grouped adjacency of triples (heads[k], labs[k], tails[k]) over Nt = B * N global nodes.

    Row u lists every distinct neighbour v of u once (a self-loop is one neighbour), ordered by (label of the pair's
    last triple, index of the pair's first triple), with that label; either direction counts.  -> dict with
    ``rowptr`` [Nt + 1], the exclusive scan of (triples with tail u) + (triples with head u), a self-loop counting in
    both (the row capacity the kernel lays out); ``len`` [Nt]; and the rows themselves, compacted: row u is
    ``nbr`` / ``lab`` [start[u], start[u + 1]).  ``key`` = row * 2^31 + label of every compacted entry, ascending."""
    h, l, t = (np.asarray(a, dtype=np.int64).reshape(-1) for a in (heads, labs, tails))
    Nt, F = B * N, len(h)
    rowptr = np.zeros(Nt + 1, dtype=np.int64)
    rowptr[1:] = np.cumsum(np.bincount(t, minlength=Nt) + np.bincount(h, minlength=Nt))
    row, nbr = np.concatenate([t, h]), np.concatenate([h, t])
    fact = np.concatenate([np.arange(F), np.arange(F)])
    pair, inv = np.unique(row * Nt + nbr, return_inverse=True)
    first = np.full(len(pair), F, dtype=np.int64)
    last = np.full(len(pair), -1, dtype=np.int64)
    np.minimum.at(first, inv.reshape(-1), fact)
    np.maximum.at(last, inv.reshape(-1), fact)
    prow, pnbr = np.divmod(pair, Nt)
    plab = l[last]
    order = np.lexsort((first, plab, prow))
    length = np.bincount(prow, minlength=Nt).astype(np.int64)
    start = np.zeros(Nt + 1, dtype=np.int64)
    start[1:] = np.cumsum(length)
    return dict(Nt=Nt, rowptr=rowptr, len=length, start=start, nbr=pnbr[order], lab=plab[order],
                key=prow[order] * _LAB + plab[order])


def row(adj, u):
    """Row u as a list of (neighbour, label)."""
    s, e = int(adj["start"][u]), int(adj["start"][u + 1])
    return list(zip(adj["nbr"][s:e].tolist(), adj["lab"][s:e].tolist()))


def used_slots(adj):
    """The slots [rowptr[u], rowptr[u] + len[u]) of every row, row after row: where the kernel's nbr / lab arrays hold
    the compacted rows (the rest of each row is capacity)."""
    ln = adj["len"]
    return np.repeat(adj["rowptr"][:-1], ln) + np.arange(int(ln.sum())) - np.repeat(adj["start"][:-1], ln)


# ---- level expansion ---------------------------------------------------------------------------------------------------

def level_count(adj, rule_off, rule_len, rule_lab, level, node, job):
    """gr_rule_level_count on the frontier (node, job) at ``level``.  -> dict with ``count`` [n] (the length of the
    segment of node's row whose label is the job's rule element ``level``; 0 once the job is finished, for a node -1
    and for a label -1), ``seg_begin`` [n] (that segment's first slot in rowptr coordinates; -1 where the count is 0,
    where the kernel's value is unspecified), ``lo`` [n] (the same in compacted coordinates), ``off`` [n + 1] (the
    int64 exclusive scan, the level total at [n]), and the jobs finishing here: ``fin`` (rule length == level) with
    ``res_begin`` / ``res_count``, the run of the job-major frontier they own."""
    rule_off, rule_len, rule_lab, node, job = (np.asarray(a, dtype=np.int64).reshape(-1)
                                               for a in (rule_off, rule_len, rule_lab, node, job))
    n = len(node)
    live = (level < rule_len[job]) & (node >= 0)
    lab = np.full(n, -1, dtype=np.int64)
    lab[live] = rule_lab[rule_off[job[live]] + level]
    live &= lab >= 0
    u = np.where(live, node, 0)
    q = u * _LAB + lab
    lo = np.searchsorted(adj["key"], q, "left")
    count = np.where(live, np.searchsorted(adj["key"], q, "right") - lo, 0)
    seg_begin = np.where(count > 0, adj["rowptr"][u] + lo - adj["start"][u], -1)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(count, out=off[1:])
    fin = np.flatnonzero(rule_len == level)
    res_begin = np.searchsorted(job, fin, "left")
    return dict(count=count, seg_begin=seg_begin, lo=lo, off=off, fin=fin, res_begin=res_begin,
                res_count=np.searchsorted(job, fin + 1, "left") - res_begin)


def level_emit(nbr, seg_begin, off, job):
    """gr_rule_level_emit: child c of the level belongs to the entry i with off[i] <= c < off[i + 1] and is
    nbr[seg_begin[i] + c - off[i]].  -> (child_node, child_parent, child_job)."""
    off = np.asarray(off, dtype=np.int64)
    parent = np.repeat(np.arange(len(off) - 1), np.diff(off))
    k = np.arange(int(off[-1])) - off[parent]
    return (np.asarray(nbr)[np.asarray(seg_begin)[parent] + k].astype(np.int64), parent,
            np.asarray(job, dtype=np.int64)[parent])


def walk_back(level_node, level_parent, rule_len, res_begin, res_count):
    """gr_rule_paths_write: job j's paths are its finishing level's entries [res_begin, + res_count), each walked back
    through the parent links into rule_len + 1 node ids, start first.  -> (paths, elem_off [J + 1])."""
    rule_len, res_begin, res_count = (np.asarray(a, dtype=np.int64) for a in (rule_len, res_begin, res_count))
    elem_off = np.zeros(len(rule_len) + 1, dtype=np.int64)
    np.cumsum(res_count * (rule_len + 1), out=elem_off[1:])
    out = np.empty(int(elem_off[-1]), dtype=np.int64)
    for j in np.flatnonzero(res_count):
        L = int(rule_len[j])
        e = res_begin[j] + np.arange(res_count[j])
        blk = np.empty((len(e), L + 1), dtype=np.int64)
        for lv in range(L, -1, -1):
            blk[:, lv] = level_node[lv][e]
            if lv:
                e = level_parent[lv][e]
        out[elem_off[j]: elem_off[j + 1]] = blk.reshape(-1)
    return out, elem_off


def expand(adj, start, rule_off, rule_len, rule_lab):
    """The level expansion of ops.rule_walks.  Job j walks from start[j] along rule_lab[rule_off[j], + rule_len[j]);
    a start of -1 with a non-empty rule is dropped (the reference finds no path), one with an empty rule is kept.

    -> dict with ``levels``: per level a dict of the frontier ``node`` / ``parent`` / ``job`` (job-major, FIFO order;
    level 0's parents are -1) and the level_count fields; per job ``res_begin`` / ``res_count`` at its finishing level;
    ``paths`` (every job's [count, len + 1] node block, job after job), ``counts`` and ``elem_off`` [J + 1]."""
    start, rule_off, rule_len, rule_lab = (np.asarray(a, dtype=np.int64).reshape(-1)
                                           for a in (start, rule_off, rule_len, rule_lab))
    J = len(start)
    keep = np.flatnonzero((rule_len == 0) | (start >= 0))
    node, job, parent = start[keep], keep, np.full(len(keep), -1, dtype=np.int64)
    res_begin, res_count = np.zeros(J, dtype=np.int64), np.zeros(J, dtype=np.int64)
    levels = []
    last = int(rule_len.max()) if J else -1
    for level in range(last + 1):
        c = level_count(adj, rule_off, rule_len, rule_lab, level, node, job)
        levels.append(dict(node=node, parent=parent, job=job, **c))
        res_begin[c["fin"]], res_count[c["fin"]] = c["res_begin"], c["res_count"]
        if level == last:
            break
        node, parent, job = level_emit(adj["nbr"], c["lo"], c["off"], job)
    paths, elem_off = walk_back([x["node"] for x in levels], [x["parent"] for x in levels], rule_len, res_begin,
                                res_count)
    return dict(levels=levels, res_begin=res_begin, res_count=res_count, paths=paths, counts=res_count,
                elem_off=elem_off)


# ---- the string level: build_graph + apply_rules ---------------------------------------------------------------------

def intern(triples):
    """Entity ids in order of first appearance (head before tail, as nx.Graph.add_edge inserts them) and label ids of
    the stripped relation strings -> (entity names, label -> id, heads, labs, tails)."""
    ent, lab2id = {}, {}
    h, l, t = [], [], []
    for a, r, b in triples:
        h.append(ent.setdefault(a, len(ent)))
        t.append(ent.setdefault(b, len(ent)))
        l.append(lab2id.setdefault(r.strip(), len(lab2id)))
    return list(ent), lab2id, np.array(h, np.int64), np.array(l, np.int64), np.array(t, np.int64)


def encode_jobs(lab2id, starts, rules):
    """(start, rule_off, rule_len, rule_lab) of the jobs; a rule element that is not a label gets -1."""
    rule_len = np.array([len(r) for r in rules], dtype=np.int64)
    rule_off = np.zeros(len(rules), dtype=np.int64)
    np.cumsum(rule_len[:-1], out=rule_off[1:])
    rule_lab = np.array([lab2id.get(x, -1) for r in rules for x in r], dtype=np.int64)
    return np.array(starts, dtype=np.int64), rule_off, rule_len, rule_lab


def apply_rules(triples, rules, sources):
    """PromptBuilder.apply_rules through ``adjacency`` and ``expand``: for every source, for every rule, the walks as
    ``[(u, rel, v), ...]`` (rel = the rule element the edge matched)."""
    names, lab2id, h, l, t = intern(triples)
    ids = {e: i for i, e in enumerate(names)}
    jobs = [(e, r) for e in sources for r in rules]
    x = expand(adjacency(h, l, t, 1, max(len(names), 1)),
               *encode_jobs(lab2id, [ids.get(e, -1) for e, _ in jobs], [r for _, r in jobs]))
    out = []
    for j, (_, r) in enumerate(jobs):
        blk = x["paths"][x["elem_off"][j]: x["elem_off"][j + 1]].reshape(-1, len(r) + 1)
        out.extend([(names[p[i]], r[i], names[p[i + 1]]) for i in range(len(r))] for p in blk.tolist())
    return out
