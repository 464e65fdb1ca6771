"""Block-wise fp64 reference of the fused joiners (DESIGN.md §14-§16) with test_gpu_joiner.py's per-element bars, for
the tests at production sizes, and a mirror of the host plan (rnnt_joiner.cu plan()).  Test infrastructure only.

joiner_reference.py and the bar helpers of test_gpu_joiner.py form whole [N, T, U, V] fp64 tensors: 2.3 GB each at
9 000 cells x V 32 000.  reference() computes the same quantities over blocks of a few thousand valid cells (pruned:
covered cells) at a time, on the inputs' device, and accumulates the gradients and their bars into fp64 [N, T, H],
[N, U, H], [V, H] and [V] outputs.  Cells no valid row stands for contribute nothing to any of them (their h is 0 in
the dense references, and their dlogits are 0), so they are skipped.  The formulas are test_gpu_joiner.py's term for
term: factor_bar, dl_error and gradient_bars, with the chunk and slab counts passed in.
"""
import types

import numpy as np
import torch

import dropout_reference as dr
import joiner_reference as jr
import pruned_joiner_reference as pjr

U_ = 2.0 ** -24

# rnnt_joiner.cu's plan() constants
TILE = 64
ALIGN = 256
SCRATCH_CAP = 256 << 20
SMS = 132
SLAB_TARGET = 2 * SMS
MAX_SLABS = 16
MAX_ROWS = 128
INT_MAX = 2 ** 31 - 1


def _up(x, a):
    return -(-x // a) * a


def plan(T, U, N, H, V, chunk_cells=None, s_range=None):
    """rnnt_joiner.cu plan() for workspace_size(T, U, N, H, V, chunk_cells, s_range): the chunk (None: the default),
    the dW slab count, the logits kernels' rows per CTA (bm), the workspace's byte offsets, and the chunk count and
    the last chunk's rows that the chunk loop runs."""
    p = types.SimpleNamespace(N=N, T=T, U=U, H=H, V=V, R=s_range)
    p.Hp, p.Vp = _up(H + 1, TILE), _up(V, TILE)
    p.cells = N * T * (U if s_range is None else s_range)
    if chunk_cells is None:   # whole waves of 128-row CTAs within the scratch cap
        row = p.Hp * 2 + p.Vp * 2 + H * 4
        wave = MAX_ROWS * SMS
        fit = SCRATCH_CAP // row
        fit = fit // wave * wave if fit >= wave else fit // MAX_ROWS * MAX_ROWS
        chunk_cells = MAX_ROWS if fit < MAX_ROWS else min(fit, INT_MAX // 2)
    p.chunk = min(chunk_cells, p.cells)
    p.rows = _up(p.chunk, MAX_ROWS)
    tiles = (p.Vp // TILE) * (p.Hp // TILE)
    p.slabs = min(-(-SLAB_TARGET // tiles), MAX_SLABS, p.rows // TILE)
    p.bm = 128 if H <= 640 else 64
    p.chunks = -(-p.cells // p.chunk)
    p.last = p.cells - (p.chunks - 1) * p.chunk
    o = 0
    for name, n in (("lse", p.cells * 4), ("denc", N * T * H * 4), ("dpred", N * U * H * 4),
                    ("dw", p.slabs * p.Vp * p.Hp * 4), ("h", p.rows * p.Hp * 2), ("dlog", p.rows * p.Vp * 2),
                    ("ds", p.rows * H * 4)):
        setattr(p, name, o)
        o = _up(o + n, ALIGN)
    p.bytes = o
    return p


def block_rows(V, budget=1 << 28):
    """Cells per block: one [rows, V] fp64 tensor within budget bytes (a block holds about eight)."""
    return max(64, budget // (8 * V))


def cells(inputs, window=None):
    """(b, t, u) int64 index tensors of the valid cells (pruned: of the cells a valid window row covers)."""
    enc, pred, _, _, _, tl, ul = inputs
    T, U = enc.shape[1], pred.shape[1]
    m = jr.masks(tl, ul, T, U)[0] if window is None else pjr.covered(window[0], window[1], tl, ul, T, U)
    return m.nonzero(as_tuple=True)


def grid_rows(inputs, c0, c1, window=None):
    """Grid rows c0 .. c1 - 1 of a call: (valid [m] bool, b, t, u [m] int64), rows dense (b, u, t) or pruned (b, r, t)
    with t fastest, u = ranges[b, t] + r; b, t, u are meaningful where valid."""
    enc, pred, _, _, _, tl, ul = inputs
    T, U = enc.shape[1], pred.shape[1]
    c = torch.arange(c0, c1, device=enc.device)
    t, bu = c % T, c // T
    if window is None:
        b, u = bu // U, bu % U
    else:
        b = bu // window[1]
        u = window[0].long()[b, t] + bu % window[1]
    valid = (t < tl.long().clamp(1, T)[b]) & (u >= 0) & (u <= ul.long().clamp(0, U - 1)[b])
    return valid, b, t, torch.where(valid, u, torch.zeros_like(u))


def keep(seed, p, b, t, u, T, U, H):
    """bool [n, H] keep mask of the cells (b, t, u): dropout_reference.keep_mask's layout, per cell."""
    c = ((b * U + u) * T + t).cpu().numpy().astype(np.uint64)[:, None]
    q = np.arange(H // 4, dtype=np.uint64)[None, :]
    words = dr.philox4x32_10((q, c, 0, 0), dr.seed_key(seed))
    x = np.stack(np.broadcast_arrays(*words), axis=-1).reshape(len(c), H)
    return torch.from_numpy(x >= np.uint64(dr.threshold(p))).to(b.device)


def terms(inputs, b, t, u, blank, activation, dpx, dpy, dropout=None):
    """fp64 quantities of the valid cells (b, t, u): h (torch's bf16 h), ht (h~ with dropout (p, seed), else h), ag
    (act' keep scale), lse, the factor bar, py, px (NaN for a label outside [0, V); -inf-free: has_label tells where
    px exists), p (softmax), gx, gy, dl and dl_err (test_gpu_joiner.dl_error)."""
    enc, pred, weight, bias, labels, tl, ul = inputs
    N, T, H = enc.shape
    U, V = pred.shape[1], weight.shape[0]
    S = U - 1
    x = types.SimpleNamespace()
    s = enc[b, t].float() + pred[b, u].float()
    x.h = (torch.tanh(s) if activation == 'tanh' else torch.relu(s)).to(torch.bfloat16)
    x.ag = jr.act_grad(x.h, activation)
    x.ht = x.h
    if dropout is not None:
        mask = keep(dropout[1], dropout[0], b, t, u, T, U, H)
        x.ht = dr.dropped_hidden(x.h, mask, dropout[0])
        x.ag = x.ag * mask.double() * dr.scale(dropout[0])
    hd, wd = x.ht.double(), weight.double()
    z = hd @ wd.T
    A = hd.abs() @ wd.abs().T
    if bias is not None:
        z = z + bias.double()
        A = A + bias.double().abs()
    x.lse = torch.logsumexp(z, -1)
    x.bar = 2 * (H + 8) * U_ * A.amax(-1) + (V / 8 + 32) * U_ + 4 * U_ * x.lse.abs()
    del A
    x.py = z[:, blank] - x.lse
    x.has_label = u < ul.long().clamp(0, S)[b]
    lbl = labels.long()[b, u.clamp(max=max(S - 1, 0))] if S > 0 else torch.zeros_like(u)
    inside = x.has_label & (lbl >= 0) & (lbl < V)
    lc = lbl.clamp(0, V - 1)
    x.px = torch.where(inside, z.gather(1, lc[:, None])[:, 0] - x.lse, torch.full_like(x.lse, float('nan')))
    x.p = torch.exp(z - x.lse[:, None])
    del z
    x.gy = dpy[b, u, t].double()
    x.gx = torch.where(x.has_label, dpx[b, u.clamp(max=max(S - 1, 0)), t].double(), torch.zeros_like(x.gy)) \
        if S > 0 else torch.zeros_like(x.gy)
    x.dl = -(x.gx + x.gy)[:, None] * x.p
    x.dl[:, blank] += x.gy
    rows = inside.nonzero(as_tuple=True)[0]
    x.dl[rows, lc[rows]] += x.gx[rows]
    x.dl_err = 2.0 ** -8 * x.dl.abs() + ((x.gx.abs() + x.gy.abs()) * 2 * x.bar)[:, None] * x.p
    return x


def reference(inputs, blank, activation, dpx, dpy, chunks, slabs, window=None, dropout=None, block=None):
    """fp64 factors, gradients and bars of a joiner call, block by block.

    dpx, dpy: the incoming gradients as the kernel gets them (only valid / covered cells are read).  chunks, slabs:
    the counts the call runs (plan()).  window: (ranges, s_range) for the pruned joiner.  dropout: (p, seed).
    Returns px [N, U-1, T], py [N, U, T] (-inf off the cells, NaN for a label outside the alphabet), lse and bar
    [N, T, U] (0 off the cells), grads (d_enc, d_pred, d_weight, d_bias) and bars, the four gradients' bars without
    the final bf16 rounding term (test_gpu_joiner.gradient_bars)."""
    enc, pred, weight, bias, labels, tl, ul = inputs
    N, T, H = enc.shape
    U, V = pred.shape[1], weight.shape[0]
    dev = enc.device
    f64 = dict(dtype=torch.float64, device=dev)
    r = types.SimpleNamespace()
    r.px = torch.full((N, U - 1, T), -float('inf'), **f64)
    r.py = torch.full((N, U, T), -float('inf'), **f64)
    r.lse = torch.zeros(N, T, U, **f64)
    r.bar = torch.zeros(N, T, U, **f64)
    de, dp, dw, db = (torch.zeros(N * T, H, **f64), torch.zeros(N * U, H, **f64), torch.zeros(V, H, **f64),
                      torch.zeros(V, **f64))
    be, bp, bw, bb = (torch.zeros_like(x) for x in (de, dp, dw, db))
    wd, wa = weight.double(), weight.double().abs()
    g_dw = (32 + N * T * U / 256 + slabs + chunks) * 2 * U_
    g_ds = (32 + V / 256) * 2 * U_
    cb, ct, cu = cells(inputs, window)
    step = block or block_rows(V)
    for i in range(0, len(cb), step):
        b, t, u = cb[i:i + step], ct[i:i + step], cu[i:i + step]
        x = terms(inputs, b, t, u, blank, activation, dpx, dpy, dropout)
        r.lse[b, t, u] = x.lse
        r.bar[b, t, u] = x.bar
        r.py[b, u, t] = x.py
        k = x.has_label.nonzero(as_tuple=True)[0]
        r.px[b[k], u[k], t[k]] = x.px[k]
        ds = (x.dl @ wd) * x.ag
        e = x.dl_err + g_ds * x.dl.abs()
        b_ds = (e @ wa) * x.ag
        del e
        de.index_add_(0, b * T + t, ds)
        dp.index_add_(0, b * U + u, ds)
        be.index_add_(0, b * T + t, b_ds + (U + chunks) * 2 * U_ * ds.abs())
        bp.index_add_(0, b * U + u, b_ds + (T + chunks) * 2 * U_ * ds.abs())
        del ds, b_ds
        hd = x.ht.double()
        dw += x.dl.T @ hd
        db += x.dl.sum(0)
        e = x.dl_err + g_dw * x.dl.abs()
        bw += e.T @ hd.abs()
        bb += e.sum(0)
        del x, e
    r.grads = (de.view(N, T, H), dp.view(N, U, H), dw, db)
    r.bars = (be.view(N, T, H), bp.view(N, U, H), bw, bb)
    return r


def gradient_ratios(got, ref, bars):
    """Worst |got - ref| / (bar + 2^-8 |ref|) of each of the four gradients (None where got is None); asserts every
    element within its bar."""
    out = []
    for name, g, r, b in zip(("d_enc", "d_pred", "d_weight", "d_bias"), got, ref, bars):
        if g is None:
            out.append(None)
            continue
        out.append(ratio(name, g, r, b + 2.0 ** -8 * r.abs()))
    return out


def ratio(name, got, ref, lim):
    """Worst |got - ref| / lim over the elements; asserts err <= lim everywhere (no floor)."""
    err = (got.to(ref.device).double() - ref).abs()
    bad = ~(err <= lim)
    assert not bad.any(), (name, int(bad.sum()), err.max().item(), (err / lim.clamp_min(1e-300)).max().item())
    nz = lim > 0
    return float((err[nz] / lim[nz]).max()) if nz.any() else 0.0
