"""Each contraction of the additive joint (rnnt_joint.cuh, rnnt_wgmma.cuh) judged alone, against float64 on the
operands the GPU itself read.

A plain joint call (rnnt_b200_add_joint_loss) runs with a caller-owned workspace; the reader below takes the
factor exponentials, the split-K slabs of S, 1/S and the weights back out of it, at the offsets carve_joint
(rnnt_entry.cu) gives them.  The float64 reference of a stage then starts from the fp32 tensors that stage read,
so the stages before it can neither hide nor cause its error:

    J1     Ef, Eg, mf, mg        from the inputs f, g
    S      the slabs of `part`   Ef . Eg^T      from the GPU's Ef, Eg;    inv_s = 1 / (sum of the slabs)
    dF     dF                    Ef * (Wm Eg) - blank / label terms      from the GPU's Ef, Eg, Wm, Bk, Lb
    dG     dG                    Eg * (Wm^T Ef) - blank / label terms    from the same

Bounds (u = 2^-24, the unit roundoff of fp32).  The contractions split every operand x into hi = x with its low 13
mantissa bits cleared and lo = x - hi (exact), so |lo| < 2^-10 |x|, and issue hi*hi + hi*lo + lo*hi per k-step.  The
tensor core reads lo as tf32 too, truncating it to 11 significant bits: an error below 2^-10 |lo| < 2^-20 |x|.
Per term x*y the products it forms therefore miss
    lo*lo  (< 2^-20 |xy|)  +  hi*(lo_y - tf32(lo_y))  (< 2^-20 |xy|)  +  (lo_x - tf32(lo_x))*hi  (< 2^-20 |xy|),
at most 3 * 2^-20 |xy|.  The accumulator is fp32 and the tensor core rounds it toward zero; every MMA into it
(three per 8 values of k) adds at most 2 ulp = 2^-22 of the running sum, and with all terms >= 0 the running sum
is at most the final one.  So a contraction over K values in one accumulator is within
    (3 * 2^-20 + 3 ceil(K / 8) * 2^-22) * sum_k |x_k y_k|
of the exact sum (dF and dG; S beyond 256 columns per slab accumulates stage-wise, with a tighter bound: s_ratio).
Everything after the accumulator is fp32 with round-to-nearest: one rounding (u) per operation, plus n u for a sum
of n + 1 terms.  No floor: a bound is relative to the magnitudes of its own terms.

    python tests/joint_stages.py SHAPE [SHAPE ...]

runs the named shapes (SHAPES) with whatever tuning hooks (RNNT_B200_*) the environment sets, and prints one JSON
line {shape: {stage: worst |error| / bound}} (inv_s in ulps): the child process of
tests/test_gpu_add_joint_stages.py.
"""
import ctypes as C
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "warp-transducer_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

ALIGN = 256          # Carver: every section starts on a 256-byte boundary
JOINT_SLICES = 16    # kJointSlices: the slab count `part` is carved for
WM_PAD = 32          # wg::kWmPad: Wm's row pitch on the fused gradient path
U24 = 2.0 ** -24

# (N, T, U, V): the training shapes, the control that passes today, and the vocabulary-tiled two-kernel shapes of
# test_gpu_add_joint_geometry
SHAPES = {
    "long": (32, 500, 151, 500),                      # two-kernel: dF K = 151 (7 stages), 4 vocabulary tiles
    "C3": (128, 150, 21, 5000),                       # fused gradient, S in 15 slabs
    "U40_T1000_long_K_dG_16_dF_tiles": (1, 1000, 40, 64),
    "V500_U73_two_kernel": (2, 136, 73, 500),         # dF K = 73 (4 stages), 3 dF tiles, 4 vocabulary tiles
    "V516_U49_two_kernel": (2, 136, 49, 516),         # dF K = 49 (3 stages), 5 vocabulary tiles, the last of 4 rows
    "V501_U151_MODE0": (2, 136, 151, 501),            # the same contractions with MODE 0 / MODE 1 operands
}


def align_up(x, a=ALIGN):
    return (x + a - 1) // a * a


def cdiv(a, b):
    return -(-a // b)


def layout(N, T, U, V):
    """carve_joint's plain sections: ({name: byte offset}, total bytes).  The base is 256-byte aligned."""
    cells, diag = N * T * U, N * (T + U - 1) * U
    sizes = [("lp2", diag * 16), ("alphas", diag * 8), ("betas", diag * 8), ("llf", N * 8), ("llb", N * 8),
             ("ef", N * T * V * 4), ("eg", N * U * V * 4), ("mf", N * T * 4), ("mg", N * U * 4),
             ("inv_s", cells * 4), ("wm", max(cells, N * T * WM_PAD) * 4), ("bk", cells * 4), ("lb", cells * 4),
             ("part", cells * 4 * JOINT_SLICES)]
    offsets, off = {}, 0
    for name, n in sizes:
        offsets[name] = off
        off = align_up(off + n)
    return offsets, off + ALIGN   # carve_joint adds one alignment's slack for an unaligned base


def workspace_size(N, T, U, V):
    from warprnnt_pytorch.joint import _lib
    n = C.c_size_t(0)
    assert _lib.rnnt_b200_add_joint_workspace_size(T, U, N, V, C.byref(n)) == 0
    return n.value


def joint_slices(V):
    """The split-K slab count the library uses at V (tuning hook included)."""
    import warprnnt_pytorch.warp_rnnt as wr
    lib = wr.lib()
    lib.rnnt_b200_debug_policy.restype = C.c_int
    lib.rnnt_b200_debug_policy.argtypes = [C.c_int, C.c_int, C.c_int]
    return lib.rnnt_b200_debug_policy(5, V, 0)


def fused_path(N, T, U):
    """run_add_joint's choice of grad_fused_kernel, under this process's tuning hooks."""
    env = os.environ
    return (U <= WM_PAD and int(env.get("RNNT_B200_JOINT_FUSED", "1")) != 0 and
            int(env.get("RNNT_B200_JOINT_SIMT", "0")) == 0 and N * T * WM_PAD < 2 ** 31)


def make_inputs(seed, N, T, U, V, blank=0):
    """Factors ~ 2 N(0, 1); ragged act_len on every third utterance from the second, ragged label_len on every
    third from the third (utterance 0 keeps both full)."""
    rng = np.random.default_rng(seed)
    tl = np.full(N, T, np.int32)
    ul = np.full(N, U - 1, np.int32)
    tl[1::3] = rng.integers(max(1, T // 2), T, size=len(tl[1::3]))
    ul[2::3] = rng.integers(0, U - 1, size=len(ul[2::3])) if U > 1 else 0
    if N == 1:
        tl[0], ul[0] = T, U - 1
    choices = np.array([k for k in range(V) if k != blank], np.int32)
    labels = rng.choice(choices, size=(N, max(U - 1, 1))).astype(np.int32)
    trans = (rng.standard_normal((N, T, V)) * 2).astype(np.float32)
    pred = (rng.standard_normal((N, U, V)) * 2).astype(np.float32)
    return trans, pred, labels, tl, ul


def run(trans, pred, labels, tl, ul, blank=0):
    """One plain loss+gradient call with a caller-owned workspace.  Returns (dF, dG, sections) as CUDA tensors;
    sections maps ef, eg, mf, mg, inv_s, wm, bk, lb to [N, rows, cols] views and part to the [slices, N, T, U]
    slabs the S contraction wrote."""
    import torch
    from warprnnt_pytorch.joint import add_joint_call
    N, T, V = trans.shape
    U = pred.shape[1]
    lab, tld, uld = (torch.as_tensor(x).cuda() for x in (labels, tl, ul))
    costs = torch.empty(N, device="cuda")
    dF = torch.full((N, T, V), float("nan"), device="cuda")
    dG = torch.full((N, U, V), float("nan"), device="cuda")
    ws = add_joint_call(torch.as_tensor(trans).cuda(), torch.as_tensor(pred).cuda(), lab, tld, uld, costs, dF, dG,
                        blank, 1.0)
    torch.cuda.synchronize()
    offsets, end = layout(N, T, U, V)
    assert ws.numel() == end == workspace_size(N, T, U, V), (ws.numel(), end)
    assert ws.data_ptr() % ALIGN == 0
    slices = joint_slices(V)
    pitch = WM_PAD if fused_path(N, T, U) else U

    def take(name, *shape):
        n = math.prod(shape)
        return ws[offsets[name]:offsets[name] + 4 * n].view(torch.float32).view(*shape)

    def logval(name, *shape):   # LogVal {int e; float l}: log2 of the value is e + l
        raw = take(name, *shape, 2)
        return raw[..., 0].view(torch.int32), raw[..., 1]

    sec = {"ef": take("ef", N, T, V), "eg": take("eg", N, U, V), "mf": take("mf", N, T), "mg": take("mg", N, U),
           "inv_s": take("inv_s", N, T, U), "wm": take("wm", N, T, pitch)[:, :, :U], "bk": take("bk", N, T, U),
           "lb": take("lb", N, T, U), "part": take("part", slices, N, T, U), "costs": costs,
           "alphas": logval("alphas", N, T, U), "betas": logval("betas", N, T, U), "llf": logval("llf", N),
           "lp2": take("lp2", N, T + U - 1, U, 4)}
    return dF, dG, sec


def _worst(err, bound):
    """max err / bound (bound > 0 everywhere it is taken; err > 0 where bound == 0 is an infinite ratio)."""
    import torch
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def j1_ratio(x, e, m, lens, add):
    """J1 of one factor: e = ex2.approx(fl(fl(x - max) * fl(log2 e))) against exp(x - max) in float64.
    fl(x - max), the fp32 log2 e and the product each move the exponent by at most u |x - max| (3 u in all), and
    ex2.approx is within 2^-21 relative; ftz flushes results below 2^-126.  m must be the row max exactly, and
    padded rows (row >= clamp(len + add, 1, R)) exactly 0 in both."""
    import torch
    N, R, V = e.shape
    worst = 0.0
    for b in range(N):
        n = min(max(int(lens[b]) + add, 1), R)
        if e[b, n:].any() or m[b, n:].any():
            return math.inf
        xb = torch.as_tensor(x[b, :n]).to(e.device)
        if not torch.equal(m[b, :n], xb.max(-1).values):
            return math.inf
        d = xb.double() - xb.max(-1, keepdim=True).values.double()
        ref = torch.exp(d)
        bound = ref * (2.0 ** -21 + 3 * U24 * d.abs()) + 2.0 ** -126
        worst = max(worst, _worst((e[b, :n].double() - ref).abs(), bound))
    return worst


def s_ratio(sec, tl, ul):
    """S = sum of the slabs (in slab order, as joint_stats_kernel) against Ef . Eg^T in float64 from the GPU's Ef
    and Eg, relative to S itself (every term >= 0).  A slab of at most 256 columns is one accumulator: the
    contraction bound, plus (slices - 1) u for the sum of the slabs.  A longer slab accumulates stage-wise
    (rnnt_wgmma.cuh Stagewise): each 32-wide k-stage of a slab is one accumulator, restarted per stage, whose 8 hi*lo / lo*hi MMAs come first (their
    running sum is below 2^-9 of the stage's, so each truncates at most 2^-22 * 2^-9 of it) and its 4 hi*hi MMAs
    last (2^-22 each); the stages add into an fp32 total (u each), the slabs in joint_stats_kernel ((slices - 1) u):
        (3 * 2^-20 + 4 * 2^-22 + 8 * 2^-31 + (stages per slab + slices - 1) u) * S.
    One accumulator over such a slab (3 ceil(K / 8) truncations) fails this bound at K = 500.
    inv_s must be 1/S rounded (1 ulp) on valid cells, 0 elsewhere.  Returns (S ratio, inv_s ratio in ulps)."""
    import torch
    part, ef, eg, inv_s = sec["part"], sec["ef"], sec["eg"], sec["inv_s"]
    slices, N, T, U = part.shape
    V = ef.shape[-1]
    kper = cdiv(cdiv(V, slices), 32) * 32      # gemm_kernel: ceil(V / slices) rounded up to its 32-wide stages
    if cdiv(V, slices) > 256:   # run_add_joint: stage-wise beyond 8 stages per slab
        rel = 3 * 2.0 ** -20 + 4 * 2.0 ** -22 + 8 * 2.0 ** -31 + (cdiv(min(kper, V), 32) + slices - 1) * U24
    else:                       # one accumulator per slab
        rel = 3 * 2.0 ** -20 + 3 * math.ceil(min(kper, V) / 8) * 2.0 ** -22 + (slices - 1) * U24
    S = part[0].clone()
    for k in range(1, slices):
        S += part[k]
    worst = ulps = 0.0
    for b in range(N):
        Tb, Ub = min(max(int(tl[b]), 1), T), min(max(int(ul[b]) + 1, 1), U)
        ref = ef[b].double() @ eg[b].double().T
        worst = max(worst, _worst((S[b, :Tb, :Ub].double() - ref[:Tb, :Ub]).abs(), rel * ref[:Tb, :Ub]))
        inv = inv_s[b]
        want = 1.0 / S[b, :Tb, :Ub]
        diff = (inv[:Tb, :Ub].view(torch.int32) - want.view(torch.int32)).abs()
        ulps = max(ulps, float(diff.max()))
        if inv[Tb:].any() or inv[:, Ub:].any():
            ulps = math.inf
    return worst, ulps


def grad_ratio(which, grad, sec, labels, tl, ul, blank, fused):
    """dF (which = 'f') or dG ('g') against the float64 product of the GPU's Ef, Eg and Wm, minus the blank and
    label terms of joint_sparse_f_kernel / joint_sparse_g_kernel from the GPU's Bk and Lb.

    Dense term Eo * sum_k Ei[k] Wm[k] (Wm >= 0, Ei >= 0): the contraction bound over the K the kernel runs (label
    positions for dF, frames for dG, zero-padded to its stage width) plus u for the epilogue's product with Eo.
    Blank and label columns: joint_sparse_*_kernel sum the terms they subtract in fp32 (strided lanes, a 5-level warp
    sum, label groups in lane order) and round once more when subtracting: n u of the dense term and the
    subtracted terms, n = ceil(K / 32) + 32 + 2."""
    import torch
    ef, eg, wm, bk, lb = (sec[k] for k in ("ef", "eg", "wm", "bk", "lb"))
    N, T, U = wm.shape
    K = U if which == "f" else T
    kpad = cdiv(K, 32 if fused else 24) * (32 if fused else 24)   # grad_fused_kernel's 32, gemm_kernel's 24
    rel = 3 * 2.0 ** -20 + 3 * math.ceil(kpad / 8) * 2.0 ** -22 + U24
    nsp = (math.ceil(K / 32) + 34) * U24
    worst = 0.0
    for b in range(N):
        Tb, Ub = min(max(int(tl[b]), 1), T), min(max(int(ul[b]) + 1, 1), U)
        W = wm[b].double()
        if which == "f":
            dense = ef[b].double() * (W @ eg[b].double())
            rows = Tb
            sp = torch.zeros_like(dense)
            sp[:, blank] += bk[b, :, :Ub].double().sum(-1)
            lab = torch.as_tensor(labels[b, :Ub - 1].astype(np.int64), device=sp.device)
            if Ub > 1:
                sp.index_add_(1, lab, lb[b, :, :Ub - 1].double())
        else:
            dense = eg[b].double() * (W.T @ ef[b].double())
            rows = Ub
            sp = torch.zeros_like(dense)
            sp[:, blank] += bk[b, :Tb].double().sum(0)
            if Ub > 1:
                u = torch.arange(Ub - 1, device=sp.device)
                lab = torch.as_tensor(labels[b, :Ub - 1].astype(np.int64), device=sp.device)
                sp[u, lab] += lb[b, :Tb, :Ub - 1].double().sum(0)
        ref = dense - sp
        g = grad[b].double()
        if g[rows:].any():
            return math.inf
        bound = rel * dense + nsp * (dense + sp)
        worst = max(worst, _worst((g[:rows] - ref[:rows]).abs(), bound[:rows]))
    return worst


def weights_ratio(sec, tl, ul):
    """joint_weights_kernel: Wm = 2^(a + b - ll) / S, Bk = 2^(a + b(t+1,u) - ll + lp_blank) (the final blank at
    (T_b - 1, U_b - 1) without b), Lb = 2^(a + b(t,u+1) - ll + lp_label), from the GPU's alphas and betas (cell-major
    LogVal: log2 = e + l), llf, lp2 (diagonal-major {m_blank, k_blank, m_label, k_label}: p = m 2^k) and inv_s,
    against float64.  The kernel forms each exponent x in fp32: integer parts exactly, then at most four roundings of
    sums of the float parts (a.l - ll.l, + b.l, + the integers, + lp) and log2f of m: |dx| <= 2 u (sum of those
    magnitudes + |x|).  exp2f adds 2 ulp, the products with inv_s and the scale one rounding each.
    Also returns the largest |Wm S - Bk - Lb| / (Wm S) over cells holding at least 2^-20 of their frame's occupancy
    (a node's occupancy is the sum of its two outgoing transitions': beta's recursion)."""
    import torch
    wm, bk, lb, inv_s = sec["wm"], sec["bk"], sec["lb"], sec["inv_s"]
    ae, al = (x.double() for x in sec["alphas"])
    be, bl = (x.double() for x in sec["betas"])
    le, ll = (x.double() for x in sec["llf"])
    N, T, U = wm.shape
    dev = wm.device
    worst = resid = 0.0
    for b in range(N):
        Tb, Ub = min(max(int(tl[b]), 1), T), min(max(int(ul[b]) + 1, 1), U)
        t = torch.arange(Tb, device=dev)[:, None]
        u = torch.arange(Ub, device=dev)[None, :]
        fac = sec["lp2"][b][t + u, u]
        lpb = fac[..., 1].view(torch.int32).double() + torch.log2(fac[..., 0].double())
        lpl = fac[..., 3].view(torch.int32).double() + torch.log2(fac[..., 2].double())
        ie, fl = ae[b, :Tb, :Ub] - le[b], al[b, :Tb, :Ub] - ll[b]          # alpha / ll: integer and float parts
        bie, bfl = be[b, :Tb, :Ub], bl[b, :Tb, :Ub]
        # successors' beta: (t+1, u) for the blank (none after the last frame but the final blank), (t, u+1) for a label
        nb_e, nb_l = torch.full_like(bie, -math.inf), torch.zeros_like(bfl)
        nb_e[:Tb - 1], nb_l[:Tb - 1] = bie[1:], bfl[1:]
        nb_e[Tb - 1, Ub - 1] = 0.0
        nl_e, nl_l = torch.full_like(bie, -math.inf), torch.zeros_like(bfl)
        nl_e[:, :Ub - 1], nl_l[:, :Ub - 1] = bie[:, 1:], bfl[:, 1:]
        for got, e, l, lp, s in ((wm[b, :Tb, :Ub], bie, bfl, 0.0, inv_s[b, :Tb, :Ub].double()),
                                 (bk[b, :Tb, :Ub], nb_e, nb_l, lpb, 1.0), (lb[b, :Tb, :Ub], nl_e, nl_l, lpl, 1.0)):
            x = ie + e + fl + l + lp
            ref = torch.exp2(x) * s
            fin = torch.isfinite(x)
            lpa = lp.abs() if torch.is_tensor(lp) else 0.0
            dx = 2 * U24 * (fl.abs() + (fl + l).abs() + (ie + e + fl + l).abs() + 2 * lpa + x.abs())
            bound = torch.where(fin, ref * (math.log(2) * dx.nan_to_num(0.0, 0.0, 0.0) + 4 * U24), 0.0) + 2.0 ** -126
            err = torch.where(fin, (got.double() - ref).abs(), got.double().abs())
            worst = max(worst, _worst(err, bound))
        gamma = wm[b, :Tb, :Ub].double() / inv_s[b, :Tb, :Ub].double()
        keep = gamma > gamma.sum(1, keepdim=True) * 2.0 ** -20
        r = ((gamma - bk[b, :Tb, :Ub].double() - lb[b, :Tb, :Ub].double()).abs() / gamma)[keep]
        resid = max(resid, float(r.max()) if r.numel() else 0.0)
    return worst, resid


def stage_ratios(N, T, U, V, seed=83, blank=0):
    """{stage: worst |error| / bound} of one call at this shape (a ratio above 1 is a failed bound)."""
    trans, pred, labels, tl, ul = make_inputs(seed, N, T, U, V, blank)
    dF, dG, sec = run(trans, pred, labels, tl, ul, blank)
    out = {"J1_f": j1_ratio(trans, sec["ef"], sec["mf"], tl, 0),
           "J1_g": j1_ratio(pred, sec["eg"], sec["mg"], ul, 1)}
    out["S"], out["inv_s_ulps"] = s_ratio(sec, tl, ul)
    fused = fused_path(N, T, U)
    out["dF"] = grad_ratio("f", dF, sec, labels, tl, ul, blank, fused)
    out["dG"] = grad_ratio("g", dG, sec, labels, tl, ul, blank, fused)
    out["W"], out["node_residual"] = weights_ratio(sec, tl, ul)
    return out


def main():
    """--slices: also report the slab count of each shape's V (the JOINT_SLICES hook's effect)."""
    names = [a for a in sys.argv[1:] if not a.startswith("--")]
    res = {name: stage_ratios(*SHAPES[name]) for name in names}
    if "--slices" in sys.argv:
        res["slices"] = {str(V): joint_slices(V) for V in sorted({SHAPES[n][3] for n in names})}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
