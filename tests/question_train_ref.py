"""Float64 restatements of the question-side training kernels (csrc/question.cu: gr_instructions_train,
gr_instructions_backward, gr_query_reform_backward) and a numpy restatement of their Philox dropout key.

``instructions_backward`` and ``reform_backward`` write out the backward by hand, in the order the kernels walk it, and
return every output the kernels write: the input gradients and the per-question weight-gradient operands.
``tests/test_question_train_host.py`` holds them to ``torch.autograd`` on the torch restatement
(``instructions_fwd`` / ``reform_fwd``) in float64.  Each also returns ``mag``: the same computation carried out on
absolute values (the softmax backward a (g_a - sum a g_a) as a (|g_a| + sum a |g_a|)), the scale of the classical
running-error bound |fl(f) - f| <= K u mag(f) for a computation of rounding depth K.  Like ``question_ref`` this does
not import ``gnn_rag_b200``.
"""
import numpy as np
import torch

F64 = torch.float64
VERY_NEG = float(torch.tensor(-100000000000.0, dtype=torch.float32))


def _d(t):
    return None if t is None else torch.as_tensor(t).to(F64)


# ---- dropout key --------------------------------------------------------------------------------------------------

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85


def philox4x32_10(key, ctr):
    """Philox4x32-10 (Salmon et al., SC'11) on uint32 numpy arrays: key = (k0, k1), ctr = (c0, c1, c2, c3), each
    broadcastable.  Returns the four output words."""
    k0, k1 = (np.asarray(k, dtype=np.uint64) for k in key)
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) for c in ctr)
    m32 = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(M0) * c0, np.uint64(M1) * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0) & m32, p1 & m32, ((p0 >> np.uint64(32)) ^ c3 ^ k1) & m32, \
            p0 & m32
        k0, k1 = (k0 + np.uint64(W0)) & m32, (k1 + np.uint64(W1)) & m32
    return c0, c1, c2, c3


def ins_keep(seed, p, b, i, site, q, c):
    """The documented key of gr_instructions_train: element (question b, step i, site, token q, column c) is kept iff
    u = (Philox4x32-10(key = seed, counter = (b, 4 i + site, q, c))[0] >> 8) * 2^-24 >= p (compared in fp32)."""
    seed = int(seed) & (2 ** 64 - 1)
    x0 = philox4x32_10((seed & 0xFFFFFFFF, seed >> 32), (b, 4 * np.asarray(i) + site, q, c))[0]
    u = (x0 >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)
    return u >= np.float32(p)


def ins_masks(seed, p, B, Q, D, I):
    """The three masks of gr_instructions_dropout_mask as bool numpy arrays: [B, I, D], [B, I, 4D], [B, I, Q, D]."""
    b, i, c = np.meshgrid(np.arange(B), np.arange(I), np.arange(D), indexing="ij")
    m0 = ins_keep(seed, p, b, i, 0, 0, c)
    b, i, c = np.meshgrid(np.arange(B), np.arange(I), np.arange(4 * D), indexing="ij")
    m1 = ins_keep(seed, p, b, i, 1, 0, c)
    b, i, q, c = np.meshgrid(np.arange(B), np.arange(I), np.arange(Q), np.arange(D), indexing="ij")
    m2 = ins_keep(seed, p, b, i, 2, q, c)
    return m0, m1, m2


# ---- instructions -------------------------------------------------------------------------------------------------

def _scaled(masks, p, dev):
    """mask / (1 - p) as float64 tensors (all ones without masks)."""
    if masks is None:
        return None
    return [torch.as_tensor(np.asarray(m), dtype=F64, device=dev) / (1.0 - p) for m in masks]


def instructions_fwd(hidden, qnode, qmask, Wq, bq, Wcq, bcq, wca, bca, masks=None, p=0.0):
    """get_instruction x I (base_encoder.py:73-114) with the three dropout sites given as masks (None = no dropout),
    torch ops in float64 (differentiable in every tensor argument).  Returns (ri [B, I, D], attn [B, I, Q])."""
    B, Q, D = hidden.shape
    s = _scaled(masks, p, hidden.device)
    ri = torch.zeros(B, D, dtype=hidden.dtype, device=hidden.device)
    outs, attns = [], []
    for i in range(len(Wq)):
        qd = qnode * s[0][:, i] if s else qnode
        q = qd @ Wq[i].t() + bq[i]
        z = torch.cat([ri, q, q - ri, q * ri], 1)
        zd = z * s[1][:, i] if s else z
        cq = zd @ Wcq.t() + bcq
        e = cq.unsqueeze(1) * hidden
        e = e * s[2][:, i] if s else e
        ca = e @ wca.reshape(-1) + bca.reshape(-1)
        attn = torch.softmax(torch.where(qmask > 0, ca, ca + VERY_NEG), 1)
        ri = (attn.unsqueeze(2) * hidden).sum(1)
        outs.append(ri)
        attns.append(attn)
    return torch.stack(outs, 1), torch.stack(attns, 1)


def instructions_backward(hidden, qnode, Wq, bq, Wcq, bcq, wca, ri, attn, grad_out, masks=None, p=0.0):
    """gr_instructions_backward in float64, given the forward's ri [B, I, D] and attn [B, I, Q] (the kernel's own, or
    those of instructions_fwd).  Returns (vals, mag): dicts with grad_hidden, grad_qnode, g_q, x_q, g_cq, x_cq, g_ca,
    x_ca (the kernel's outputs) and their absolute-value restatement."""
    hid, qn, wca = _d(hidden), _d(qnode), _d(wca).reshape(-1)
    Wq, bq, Wcq, bcq = [_d(w) for w in Wq], [_d(b) for b in bq], _d(Wcq), _d(bcq)
    ri, attn, G = _d(ri), _d(attn), _d(grad_out)
    B, Q, D = hid.shape
    I = len(Wq)
    s = _scaled(masks, p, hid.device)
    one = lambda t: torch.ones_like(t)   # noqa: E731
    out = {k: [None] * I for k in ("g_q", "x_q", "g_cq", "x_cq", "g_ca", "x_ca")}
    mag = {k: [None] * I for k in out}
    gh, mgh = torch.zeros_like(hid), torch.zeros_like(hid)
    gqn, mgqn = torch.zeros_like(qn), torch.zeros_like(qn)
    gr, mgr = G[:, I - 1], G[:, I - 1].abs()
    for i in range(I - 1, -1, -1):
        s0 = s[0][:, i] if s else one(qn)
        s1 = s[1][:, i] if s else torch.ones(B, 4 * D, dtype=F64, device=hid.device)
        s2 = s[2][:, i] if s else one(hid)
        rp = ri[:, i - 1] if i > 0 else torch.zeros_like(qn)
        a = attn[:, i]
        qd = qn * s0
        q = qd @ Wq[i].t() + bq[i]
        mq = qd.abs() @ Wq[i].abs().t() + bq[i].abs()
        zd = torch.cat([rp, q, q - rp, q * rp], 1) * s1
        mzd = torch.cat([rp.abs(), mq, mq + rp.abs(), mq * rp.abs()], 1) * s1
        cq = zd @ Wcq.t() + bcq
        mcq = mzd @ Wcq.abs().t() + bcq.abs()
        e = cq.unsqueeze(1) * hid * s2
        me = mcq.unsqueeze(1) * hid.abs() * s2
        ga = (hid * gr.unsqueeze(1)).sum(2)                                  # dattn
        mga = (hid.abs() * mgr.unsqueeze(1)).sum(2)
        gca = a * (ga - (a * ga).sum(1, keepdim=True))
        mgca = a * (mga + (a * mga).sum(1, keepdim=True))
        ge = gca.unsqueeze(2) * wca * s2                                     # dL/d(cq * hidden) after the mask
        mge = mgca.unsqueeze(2) * wca.abs() * s2
        gh = gh + a.unsqueeze(2) * gr.unsqueeze(1) + ge * cq.unsqueeze(1)
        mgh = mgh + a.unsqueeze(2) * mgr.unsqueeze(1) + mge * mcq.unsqueeze(1)
        gcq = (ge * hid).sum(1)
        mgcq = (mge * hid.abs()).sum(1)
        gz = (gcq @ Wcq) * s1
        mgz = (mgcq @ Wcq.abs()) * s1
        g0, g1, g2, g3 = gz.split(D, 1)
        m0, m1, m2, m3 = mgz.split(D, 1)
        gq = g1 + g2 + g3 * rp
        mgq = m1 + m2 + m3 * rp.abs()
        gri = g0 - g2 + g3 * q
        mgri = m0 + m2 + m3 * mq
        gqn = gqn + (gq @ Wq[i]) * s0
        mgqn = mgqn + (mgq @ Wq[i].abs()) * s0
        for k, v, m in (("g_q", gq, mgq), ("x_q", qd, qd.abs()), ("g_cq", gcq, mgcq), ("x_cq", zd, mzd),
                        ("g_ca", gca, mgca), ("x_ca", e, me)):
            out[k][i], mag[k][i] = v, m
        if i > 0:
            gr, mgr = G[:, i - 1] + gri, G[:, i - 1].abs() + mgri
    vals = {k: torch.stack(v, 1) for k, v in out.items()}
    mags = {k: torch.stack(v, 1) for k, v in mag.items()}
    vals.update(grad_hidden=gh, grad_qnode=gqn)
    mags.update(grad_hidden=mgh, grad_qnode=mgqn)
    return vals, mags


# ---- query reform -------------------------------------------------------------------------------------------------

def reform_fwd(seed, h, ins, Wr, Wg, B, N):
    """QueryReform + Fusion for every instruction (query_update.py:6-44) as differentiable float64 torch ops.
    seed [B, N], h [B*N, D], ins [B, I, D].  Returns [B, I, D]."""
    y = torch.bmm(seed.view(B, 1, N), h.reshape(B, N, -1)).squeeze(1)
    outs = []
    for j in range(ins.shape[1]):
        x = ins[:, j]
        z = torch.cat([x, y, x - y], 1)
        g = torch.sigmoid(z @ Wg[j].t())
        outs.append(g * (z @ Wr[j].t()) + (1 - g) * x)
    return torch.stack(outs, 1)


def reform_backward(seed, h, ins, Wr, Wg, B, N, grad_out):
    """gr_query_reform_backward in float64.  Returns dict(grad_ins, grad_h [B*N, D] (zero off the seed rows), g_r, g_g,
    x_z, y, r, g) -- y, r and g for the callers' bounds."""
    s, x, G = _d(seed), _d(ins), _d(grad_out)
    H = _d(h).reshape(B * N, -1)
    y = torch.bmm(s.view(B, 1, N), H.view(B, N, -1)).squeeze(1)
    I = x.shape[1]
    out = {k: [] for k in ("grad_ins", "g_r", "g_g", "x_z", "r", "g")}
    gy = torch.zeros_like(y)
    for j in range(I):
        xj, Wrj, Wgj = x[:, j], _d(Wr[j]), _d(Wg[j])
        z = torch.cat([xj, y, xj - y], 1)
        r, g = z @ Wrj.t(), torch.sigmoid(z @ Wgj.t())
        gr = G[:, j] * g
        gg = G[:, j] * (r - xj) * g * (1 - g)
        gz = gr @ Wrj + gg @ Wgj
        D = xj.shape[1]
        out["grad_ins"].append(G[:, j] * (1 - g) + gz[:, :D] + gz[:, 2 * D:])
        gy = gy + gz[:, D:2 * D] - gz[:, 2 * D:]
        for k, v in (("g_r", gr), ("g_g", gg), ("x_z", z), ("r", r), ("g", g)):
            out[k].append(v)
    res = {k: torch.stack(v, 1) for k, v in out.items()}
    res["grad_h"] = (s.view(B, N, 1) * gy.view(B, 1, -1)).reshape(B * N, -1)
    res["y"], res["grad_y"] = y, gy
    return res
