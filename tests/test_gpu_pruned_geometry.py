"""Pruned RNN-T loss (DESIGN.md §8) at the boundaries of its streaming-kernel dispatch (rnnt_entry.cu stream_pass,
stream_passes, chunk_pass) in every storage type, with the gradient options, at the window edges, on the multi-warp
lattice wavefronts and in the grouped schedule, against the fp64 reference (tests/pruned_reference.py).

Every shape asserts, from a torch.profiler CUDA trace, the PRUNED instantiation (last template argument true) of the
pass-1 and pass-2 kernels it names, so the table cannot drift from the dispatch:

    chunk   rowstats / grad_chunk_kernel<T, TPR, NT, ...>: rows of <= 512 B (fp32 V <= 128, fp64 V <= 64) and 16-byte
            aligned logits.  NT / TPR rows per chunk (fp32 NT = 256, fp64 128), staged with one bulk copy unless the
            chunk's byte count is not a multiple of 16 (a ragged last chunk: scalar loads and stores)
    tile    rowstats / grad_tile_kernel<T, VEC, LPR, ...>: nv = V / VEC <= 256 vectors, LPR = the fewest lanes >= 2
            with 8 * LPR >= nv
    row     rowstats / grad_row_kernel<T, VEC, NV, ...>: nv > 256, one CTA per row (256 threads, 128 for 16-bit
            storage), NV vectors per thread per trip: ceil(nv / threads) up to 6, else 8, for 16-byte vectors of 4- and
            2-byte storage; else 2 / 4 / 8
    VEC     the widest of 16 / sizeof(storage), 2 (fp32 only) and 1 that the base addresses and the row pitch allow

Tolerances: costs rtol 1e-5 (fp32 arithmetic: fp32, bf16, fp16) / 1e-11 (fp64); gradients |g - g_ref| <= rel |g_ref|
+ floor with (1e-4, 1e-6) for fp32, (1e-9, 1e-12) for fp64 and (2 eps, 1e-6) for 16-bit storage, where the reference
runs on the rounded logits.  Every call starts from a gradient full of NaN; padding rows must come out as exact zeros,
and an utterance without a path as cost +inf with an all-zero gradient.
"""
import time
import warnings

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from pruned_reference import pruned_loss, random_monotone_ranges
from test_gpu_pruned import padding_mask
from test_gpu_tuning_hooks import norm

pytestmark = pytest.mark.gpu

DTYPE = {"fp32": torch.float32, "fp64": torch.float64, "bf16": torch.bfloat16, "fp16": torch.float16}
CODE = {"fp32": 0, "bf16": 1, "fp16": 2, "fp64": 3}
ARITH = {"fp32": "float", "fp64": "double", "bf16": "float", "fp16": "float"}
IO = {"fp32": "float", "fp64": "double", "bf16": "__nv_bfloat16", "fp16": "__half"}
EPS16 = {"bf16": 2.0 ** -8, "fp16": 2.0 ** -11}

# name: (storage, (N, T, U, V, R, blank), (kernel family, TPR / VEC, NT / LPR / NV)).  N >= 3 everywhere, so that
# windows() leaves one utterance without a path.
SHAPES = {
    # fp32 chunk kernels, NT = 256 threads: TPR = 1 (V <= 32 odd, V <= 16 even), 2 (even V <= 64), 4 (V <= 128)
    "fp32_chunk_TPR1_V31_one_ragged_chunk": ("fp32", (3, 7, 5, 31, 3, 0), ("chunk", 1, 256)),   # 63 rows, not bulk
    "fp32_chunk_TPR1_V5_straddling_ragged_last": ("fp32", (5, 37, 8, 5, 3, 4), ("chunk", 1, 256)),   # 555 rows:
    #   chunks of 256, 256 and 43 rows (43 * 5 * 4 B, not bulk); 256 % R != 0, so frames straddle the boundaries
    "fp32_chunk_TPR1_V7_all_padding_chunk": ("fp32", (3, 200, 6, 7, 3, 0), ("chunk", 1, 256)),   # PADDED below:
    #   rows 600..1199 are padding, chunk 3 (rows 768..1023) holds nothing else in either pass; 8 chunks in all
    "fp32_chunk_TPR1_V16_pairs": ("fp32", (3, 9, 5, 16, 2, 0), ("chunk", 1, 256)),
    "fp32_chunk_TPR2_V50_two_chunks": ("fp32", (4, 20, 6, 50, 3, 0), ("chunk", 2, 256)),   # 128 + 112 rows
    "fp32_chunk_TPR4_V100": ("fp32", (3, 11, 5, 100, 3, 7), ("chunk", 4, 256)),             # 64 + 35 rows
    "fp32_chunk_TPR4_V128_longest_row": ("fp32", (3, 8, 5, 128, 4, 0), ("chunk", 4, 256)),  # 512 B rows
    # fp32 register tiles (rows > 512 B)
    "fp32_tile_VEC4_LPR8_V256": ("fp32", (3, 6, 4, 256, 3, 0), ("tile", 4, 8)),      # nv 64: 8 lanes x 8, full
    "fp32_tile_VEC4_LPR16_V260": ("fp32", (3, 6, 4, 260, 3, 5), ("tile", 4, 16)),    # nv 65
    "fp32_tile_VEC4_LPR32_V1024": ("fp32", (3, 5, 4, 1024, 3, 0), ("tile", 4, 32)),  # nv 256, the last tile
    "fp32_tile_VEC2_LPR16_V130": ("fp32", (3, 6, 4, 130, 3, 0), ("tile", 2, 16)),    # nv 65
    "fp32_tile_VEC2_LPR32_V510": ("fp32", (3, 6, 4, 510, 3, 1), ("tile", 2, 32)),    # nv 255
    "fp32_tile_VEC1_LPR32_V129": ("fp32", (3, 6, 4, 129, 3, 0), ("tile", 1, 32)),    # first odd V past the chunks
    "fp32_tile_VEC1_LPR32_V255": ("fp32", (3, 5, 3, 255, 2, 0), ("tile", 1, 32)),
    # fp32 CTA per row, 16-byte fast path: NV = ceil(V / 4 / 256) exactly, up to 6
    "fp32_row_VEC4_NV2_V1028": ("fp32", (3, 4, 3, 1028, 3, 5), ("row", 4, 2)),
    "fp32_row_VEC4_NV3_V3000": ("fp32", (3, 4, 3, 3000, 2, 0), ("row", 4, 3)),
    "fp32_row_VEC4_NV4_V4096": ("fp32", (3, 4, 3, 4096, 2, 0), ("row", 4, 4)),
    "fp32_row_VEC4_NV5_V5000": ("fp32", (3, 5, 4, 5000, 3, 0), ("row", 4, 5)),   # the C3 benchmark's kernel
    "fp32_row_VEC4_NV6_V6000": ("fp32", (3, 4, 3, 6000, 2, 7), ("row", 4, 6)),
    "fp32_row_VEC4_NV8_V8192_one_trip": ("fp32", (3, 4, 3, 8192, 2, 0), ("row", 4, 8)),
    "fp32_row_VEC4_NV8_V10000_two_trips": ("fp32", (3, 4, 3, 10000, 2, 0), ("row", 4, 8)),
    # fp32 CTA per row, generic: NV 2 / 4 / 8
    "fp32_row_VEC2_NV2_V514": ("fp32", (3, 4, 3, 514, 2, 0), ("row", 2, 2)),
    "fp32_row_VEC2_NV4_V1030": ("fp32", (3, 4, 3, 1030, 3, 0), ("row", 2, 4)),
    "fp32_row_VEC2_NV8_V5002_two_trips": ("fp32", (3, 4, 3, 5002, 2, 0), ("row", 2, 8)),
    "fp32_row_VEC1_NV2_V257": ("fp32", (3, 5, 3, 257, 3, 0), ("row", 1, 2)),
    "fp32_row_VEC1_NV8_V4001_two_trips": ("fp32", (3, 4, 3, 4001, 2, 0), ("row", 1, 8)),
    # fp64: chunk kernels with NT = 128 (V <= 64), register tiles and CTA per row at VEC 2 (even V) / 1
    "fp64_chunk_TPR1_V5_one_ragged_chunk": ("fp64", (3, 7, 5, 5, 3, 0), ("chunk", 1, 128)),   # 63 rows, not bulk
    "fp64_chunk_TPR2_V33_straddling_ragged_last": ("fp64", (3, 29, 6, 33, 3, 0), ("chunk", 2, 128)),   # 261 rows:
    #   4 chunks of 64 and one of 5 (5 * 33 * 8 B, not bulk)
    "fp64_chunk_TPR2_V64": ("fp64", (3, 9, 5, 64, 4, 0), ("chunk", 2, 128)),
    "fp64_tile_VEC1_LPR16_V65": ("fp64", (3, 6, 4, 65, 3, 0), ("tile", 1, 16)),
    "fp64_tile_VEC2_LPR8_V100": ("fp64", (3, 6, 4, 100, 3, 0), ("tile", 2, 8)),
    "fp64_tile_VEC2_LPR32_V512": ("fp64", (3, 5, 3, 512, 2, 0), ("tile", 2, 32)),
    "fp64_row_VEC2_NV2_V514": ("fp64", (3, 4, 3, 514, 2, 0), ("row", 2, 2)),
    "fp64_row_VEC2_NV4_V1030": ("fp64", (3, 4, 3, 1030, 3, 0), ("row", 2, 4)),
    "fp64_row_VEC1_NV4_V601": ("fp64", (3, 4, 3, 601, 3, 0), ("row", 1, 4)),
    "fp64_row_VEC1_NV8_V2049_two_trips": ("fp64", (3, 4, 3, 2049, 2, 0), ("row", 1, 8)),
    # lattice wavefronts fed mostly log-zero factors (LATTICE below): fp32 multi-warp (maxU > 64, factor ring of 8
    # diagonals), fp64 multi-warp log domain (maxU > 32)
    "fp32_lattice_U65_R4": ("fp32", (3, 40, 65, 20, 4, 0), ("chunk", 2, 256)),
    "fp32_lattice_U65_R8": ("fp32", (3, 20, 65, 20, 8, 0), ("chunk", 2, 256)),
    "fp32_lattice_U301_R4": ("fp32", (3, 120, 301, 12, 4, 0), ("chunk", 1, 256)),
    "fp32_lattice_U301_R8": ("fp32", (3, 60, 301, 12, 8, 0), ("chunk", 1, 256)),
    "fp64_lattice_U40_R4": ("fp64", (3, 30, 40, 12, 4, 0), ("chunk", 1, 128)),
    "fp64_lattice_U150_R8": ("fp64", (3, 30, 150, 12, 8, 0), ("chunk", 1, 128)),
}
# 16-bit storage (fp32 arithmetic, never the chunk kernels): tiles at every LPR, rows at every exact NV, and VEC 1
for _s in ("bf16", "fp16"):
    SHAPES.update({
        _s + "_tile_VEC8_LPR2_V64": (_s, (3, 6, 4, 64, 3, 0), ("tile", 8, 2)),
        _s + "_tile_VEC8_LPR4_V256": (_s, (3, 6, 4, 256, 3, 1), ("tile", 8, 4)),
        _s + "_tile_VEC8_LPR8_V512": (_s, (3, 6, 4, 512, 3, 0), ("tile", 8, 8)),
        _s + "_tile_VEC8_LPR16_V1024": (_s, (3, 5, 4, 1024, 3, 0), ("tile", 8, 16)),
        _s + "_tile_VEC8_LPR32_V2048": (_s, (3, 5, 3, 2048, 2, 0), ("tile", 8, 32)),
        _s + "_tile_VEC1_LPR8_V37": (_s, (3, 6, 4, 37, 3, 0), ("tile", 1, 8)),
        _s + "_row_VEC8_NV3_V3000": (_s, (3, 4, 3, 3000, 2, 0), ("row", 8, 3)),
        _s + "_row_VEC8_NV4_V4096": (_s, (3, 4, 3, 4096, 2, 0), ("row", 8, 4)),
        _s + "_row_VEC8_NV5_V5000": (_s, (3, 5, 4, 5000, 3, 0), ("row", 8, 5)),
        _s + "_row_VEC8_NV6_V6000": (_s, (3, 4, 3, 6000, 2, 5), ("row", 8, 6)),
        _s + "_row_VEC8_NV8_V8192": (_s, (3, 4, 3, 8192, 2, 0), ("row", 8, 8)),
        _s + "_row_VEC8_NV8_V10000_two_trips": (_s, (3, 4, 3, 10000, 2, 0), ("row", 8, 8)),
        _s + "_row_VEC1_NV8_V5001": (_s, (3, 4, 3, 5001, 2, 0), ("row", 1, 8)),
    })
# the utterance whose every window starts past its U_b (all its rows padding)
PADDED = {"fp32_chunk_TPR1_V7_all_padding_chunk": 1}
# the lattice kernel a shape must also launch
LATTICE = {
    "fp32_lattice_U65_R4": "lattice_lin_kernel<1, true, 8>",
    "fp32_lattice_U65_R8": "lattice_lin_kernel<1, true, 8>",
    "fp32_lattice_U301_R4": "lattice_lin_kernel<1, true, 8>",
    "fp32_lattice_U301_R8": "lattice_lin_kernel<1, true, 8>",
    "fp64_lattice_U40_R4": "lattice_kernel<double, true>",
    "fp64_lattice_U150_R8": "lattice_kernel<double, true>",
}


@pytest.fixture(scope="module")
def wr():
    import warprnnt_pytorch.warp_rnnt as wr
    import warprnnt_pytorch.pruned   # noqa: F401  (argtypes of the pruned entries)
    return wr


def heads(storage, family, a, b, scaled=False, reg=False):
    """The template heads of the PRUNED pass-1 and pass-2 kernels of `family` with parameters (a, b)."""
    t, io, s, r = ARITH[storage], IO[storage], str(scaled).lower(), str(reg).lower()
    if family == "chunk":
        return ("rowstats_chunk_kernel<%s, %d, %d, true>" % (t, a, b),
                "grad_chunk_kernel<%s, %d, %d, %s, %s, true>" % (t, a, b, s, r))
    return ("rowstats_%s_kernel<%s, %d, %d, %s, true>" % (family, t, a, b, io),
            "grad_%s_kernel<%s, %d, %d, %s, %s, %s, true>" % (family, t, a, b, s, io, r))


def assert_launched(kernels, *names):
    for name in names:
        assert any(name in k for k in kernels), (name, sorted(k for k in kernels if "b200rnnt" in k))


def make(name, storage, N, T, U, V, R, blank):
    """(rng, logits [N,T,R,V] float64 as the kernels see them, labels, act_lens, label_lens)."""
    rng = np.random.default_rng(sum(map(ord, name)))
    choices = np.array([k for k in range(V) if k != blank], np.int32)
    labels = rng.choice(choices, size=(N, max(U - 1, 1))).astype(np.int32)
    tl = rng.integers(max(1, T // 2), T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0] = T, U - 1
    logits = rng.standard_normal((N, T, R, V)) * 2
    if storage in EPS16:   # the reference sees the rounded logits
        logits = torch.tensor(logits).to(DTYPE[storage]).double().numpy()
    return rng, logits, labels, tl, ul


def windows(rng, tl, ul, T, R, padded=None):
    """random_monotone_ranges, then: utterance 1's first window starts at -1 and its frames past T_b at the int32
    extremes; the last utterance's middle frame starts past U_b (no path); every window of `padded` past U_b."""
    s = random_monotone_ranges(rng, tl, ul, T, R).astype(np.int64)
    N = len(tl)
    s[1, 0] = -1
    s[1, tl[1]:] = np.where(np.arange(T - tl[1]) % 2, -2 ** 31, 2 ** 31 - 1)
    if N >= 3:
        s[N - 1, tl[N - 1] // 2] = ul[N - 1] + 1
    if padded is not None:
        s[padded] = ul[padded] + 1 + np.arange(T)
    return s.astype(np.int32)


def profiled(call, attempts=6):
    """(call(), the normalised names of the CUDA kernels it ran) from a torch.profiler trace.  On an H100 the trace
    of such a short session has now and then come back without any device activity, even for the fill kernels of
    the call's own outputs, several sessions in a row.  A call whose trace is empty therefore runs again after a
    pause, so that a missing trace is not taken for a missing kernel.  `call` resets its own outputs."""
    for k in range(attempts):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            out = call()
            torch.cuda.synchronize()
        kernels = {norm(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if kernels:
            return out, kernels
        warnings.warn("torch.profiler returned a trace without CUDA activity; running the call again")
        time.sleep(0.5 * (k + 1))
    raise AssertionError("torch.profiler recorded no CUDA activity in %d sessions" % attempts)


def run(wr, storage, logits, ranges, labels, tl, ul, U, blank, lam=0.0, clamp=-1.0, grad_costs=None, grad_scale=1.0,
        offset=0):
    """One profiled pruned call: (costs, gradient as float64, kernel names, launches).  grad_costs given:
    rnnt_b200_pruned_forward then rnnt_b200_pruned_backward_ex with those per-utterance multipliers and grad_scale
    (the operator's split); else the full call rnnt_b200_pruned_loss_async_ex.  offset: the logits and the gradient
    are contiguous views `offset` elements into larger buffers."""
    from warprnnt_pytorch.pruned import pruned_workspace_size
    N, T, R, V = logits.shape
    dt = DTYPE[storage]
    cdt = torch.float64 if storage == "fp64" else torch.float32
    n = logits.size
    x = torch.zeros(n + offset, dtype=dt, device="cuda")[offset:].view(N, T, R, V)
    x.copy_(torch.as_tensor(logits))
    g = torch.full((n + offset,), float("nan"), dtype=dt, device="cuda")[offset:].view(N, T, R, V)
    rg, lab, tld, uld = (torch.as_tensor(np.ascontiguousarray(a)).cuda() for a in (ranges, labels, tl, ul))
    costs = torch.full((N,), float("nan"), dtype=cdt, device="cuda")
    ws = torch.empty(pruned_workspace_size(T, U, R, N, 8 if storage == "fp64" else 4), dtype=torch.uint8,
                     device="cuda")
    opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream().cuda_stream, blank_label=blank,
                         maxT=T, maxU=U, batch_first=True)
    gopt = wr.rnntGradOptions(lam, max(clamp, 0.0))
    lib = wr.lib()

    def call():
        g.fill_(float("nan"))
        costs.fill_(float("nan"))
        if grad_costs is None:
            st = lib.rnnt_b200_pruned_loss_async_ex(CODE[storage], 0, x.data_ptr(), g.data_ptr(), rg.data_ptr(), R,
                                                    lab.data_ptr(), uld.data_ptr(), tld.data_ptr(), V, N,
                                                    costs.data_ptr(), 1.0, gopt, ws.data_ptr(), opt)
            assert st == 0, wr.status_string(st)
            return wr.last_launch_count()
        gc = torch.as_tensor(grad_costs, dtype=cdt).cuda()
        st = lib.rnnt_b200_pruned_forward(CODE[storage], x.data_ptr(), rg.data_ptr(), R, lab.data_ptr(),
                                          uld.data_ptr(), tld.data_ptr(), V, N, costs.data_ptr(), 1, ws.data_ptr(), opt)
        assert st == 0, wr.status_string(st)
        launches = wr.last_launch_count()
        st = lib.rnnt_b200_pruned_backward_ex(CODE[storage], x.data_ptr(), g.data_ptr(), rg.data_ptr(), R,
                                              lab.data_ptr(), uld.data_ptr(), tld.data_ptr(), V, N, gc.data_ptr(),
                                              grad_scale, gopt, ws.data_ptr(), opt)
        assert st == 0, wr.status_string(st)
        return launches + wr.last_launch_count()

    launches, kernels = profiled(call)
    return costs.cpu().numpy().astype(np.float64), g.double().cpu().numpy(), kernels, launches


def tolerance(storage):
    """(cost rtol, gradient rel, gradient floor)."""
    if storage == "fp64":
        return 1e-11, 1e-9, 1e-12
    if storage in EPS16:
        return 1e-5, 2 * EPS16[storage], 1e-6
    return 1e-5, 1e-4, 1e-6


def check(storage, costs, g, logits, ranges, labels, tl, ul, blank, lam=0.0, clamp=-1.0, scale=None):
    """costs and gradient against pruned_loss on the same logits (scale: per-utterance gradient multipliers); the
    padding rows exact zeros; no path: +inf and an all-zero gradient.  Returns the reference costs."""
    c_ref, g_ref = pruned_loss(logits, labels, tl, ul, ranges, blank, lam, clamp)
    if scale is not None:
        g_ref = g_ref * np.asarray(scale, np.float64)[:, None, None, None]
    assert not np.isnan(g).any(), "gradient elements left undefined"
    fin = np.isfinite(c_ref)
    assert (costs[~fin] == np.inf).all() and np.isfinite(costs[fin]).all(), (costs, c_ref)
    rtol, rel, floor = tolerance(storage)
    assert np.allclose(costs[fin], c_ref[fin], rtol=rtol, atol=0), (costs, c_ref)
    excess = np.abs(g - g_ref) - (rel * np.abs(g_ref) + floor)
    assert (excess <= 0).all(), "max |g - g_ref| %.3g, worst excess %.3g at %s" % (
        np.abs(g - g_ref).max(), excess.max(), np.unravel_index(np.argmax(excess), g.shape))
    assert not g[padding_mask(ranges, tl, ul, logits.shape[2])].any(), "padding rows not zero"
    assert not g[~fin].any(), "an utterance without a path has a gradient"
    return c_ref


@pytest.mark.parametrize("name", list(SHAPES))
def test_pruned_boundary_shape(wr, name):
    storage, (N, T, U, V, R, blank), (family, a, b) = SHAPES[name]
    rng, logits, labels, tl, ul = make(name, storage, N, T, U, V, R, blank)
    ranges = windows(rng, tl, ul, T, R, PADDED.get(name))
    costs, g, kernels, launches = run(wr, storage, logits, ranges, labels, tl, ul, U, blank)
    assert_launched(kernels, *heads(storage, family, a, b), "lattice_fill_kernel<%s>" % ARITH[storage])
    if name in LATTICE:
        assert_launched(kernels, LATTICE[name])
    assert launches == 4   # the log-zero fill, pass 1, the lattice, pass 2
    c_ref = check(storage, costs, g, logits, ranges, labels, tl, ul, blank)
    assert np.isfinite(c_ref).any() and np.isinf(c_ref[N - 1])


def clamp_for(logits, labels, tl, ul, ranges, blank, lam):
    """A float32 clamp that clips about 3 % of the non-zero FastEmit gradient elements."""
    _, g = pruned_loss(logits, labels, tl, ul, ranges, blank, lam)
    return float(np.float32(np.quantile(np.abs(g[g != 0]), 0.97)))


# one shape per kernel family and storage type, with per-utterance scales (SCALED) x FastEmit and clamp (REG)
OPTION_SHAPES = ["fp32_chunk_TPR2_V50_two_chunks", "fp32_chunk_TPR1_V5_straddling_ragged_last",
                 "fp32_tile_VEC4_LPR16_V260", "fp32_tile_VEC1_LPR32_V129", "fp32_row_VEC4_NV5_V5000",
                 "fp32_row_VEC2_NV4_V1030", "fp64_chunk_TPR2_V33_straddling_ragged_last", "fp64_tile_VEC2_LPR8_V100",
                 "fp64_row_VEC1_NV4_V601", "bf16_tile_VEC8_LPR16_V1024", "bf16_row_VEC8_NV5_V5000",
                 "fp16_tile_VEC8_LPR4_V256", "fp16_row_VEC8_NV3_V3000"]


@pytest.mark.parametrize("name", OPTION_SHAPES)
def test_scaled_and_gradient_options(wr, name):
    """plain; grad_costs (distinct per utterance) x grad_scale 0.75 through the split backward; FastEmit 0.5 with a
    clamp that clips ~3 % of the elements; both.  Each runs the (SCALED, REG) instantiation of its family."""
    storage, (N, T, U, V, R, blank), (family, a, b) = SHAPES[name]
    rng, logits, labels, tl, ul = make(name, storage, N, T, U, V, R, blank)
    ranges = windows(rng, tl, ul, T, R)
    lam = 0.5
    clamp = clamp_for(logits, labels, tl, ul, ranges, blank, lam)
    grad_costs = np.linspace(0.5, 2.0, N)
    scale = 0.75 * grad_costs
    for scaled in (False, True):
        for reg in (False, True):
            kw = dict(lam=lam, clamp=clamp) if reg else {}
            sc = dict(grad_costs=grad_costs, grad_scale=0.75) if scaled else {}
            costs, g, kernels, _ = run(wr, storage, logits, ranges, labels, tl, ul, U, blank, **kw, **sc)
            assert_launched(kernels, *heads(storage, family, a, b, scaled, reg))
            check(storage, costs, g, logits, ranges, labels, tl, ul, blank, scale=scale if scaled else None, **kw)
    assert 0 < clamp < np.inf


# ---- window edges ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", ["fp32", "fp64"])
@pytest.mark.parametrize("V", [50, 1030])
def test_one_row_per_frame(wr, storage, V):
    """R = 1: a path exists only where U_b = 1 (every label position needs a window of its own)."""
    N, T, U, R = 5, 6, 4, 1
    rng, logits, labels, tl, ul = make("R1", storage, N, T, U, V, R, 0)
    ul[:] = [0, 2, 0, 3, 0]
    ranges = random_monotone_ranges(rng, tl, ul, T, R)
    costs, g, _, _ = run(wr, storage, logits, ranges, labels, tl, ul, U, 0, lam=0.5)
    fin = np.isfinite(check(storage, costs, g, logits, ranges, labels, tl, ul, 0, lam=0.5))
    assert np.array_equal(fin, ul == 0)


@pytest.mark.parametrize("storage", ["fp32", "fp64", "bf16"])
@pytest.mark.parametrize("extra", [0, 3], ids=["R_eq_maxU", "R_gt_maxU"])
def test_windows_as_wide_as_the_lattice(wr, storage, extra):
    """R = maxU and R > maxU with non-decreasing starts from <= 0 up to U_b - 1: every utterance keeps a path, and the
    rows below u = 0 or at u >= U_b are padding."""
    N, T, U, V = 4, 7, 6, 40
    R = U + extra
    rng, logits, labels, tl, ul = make("wide%d" % extra, storage, N, T, U, V, R, 0)
    ranges = np.zeros((N, T), np.int32)
    for b in range(N):
        s = np.sort(rng.integers(-extra, ul[b] + 1, size=T))
        s[0] = min(s[0], 0)
        ranges[b] = s
    assert ranges.any()
    costs, g, _, _ = run(wr, storage, logits, ranges, labels, tl, ul, U, 0)
    assert np.isfinite(check(storage, costs, g, logits, ranges, labels, tl, ul, 0)).all()


@pytest.mark.parametrize("storage", ["fp32", "fp64", "fp16"])
def test_single_frame(wr, storage):
    """T = 1: every label is emitted in frame 0, so a path exists exactly where U_b <= R."""
    N, T, U, V, R = 4, 1, 5, 300, 3
    rng, logits, labels, tl, ul = make("T1", storage, N, T, U, V, R, 0)
    ul[:] = [4, 2, 0, 1]
    ranges = np.zeros((N, T), np.int32)
    costs, g, _, _ = run(wr, storage, logits, ranges, labels, tl, ul, U, 0)
    fin = np.isfinite(check(storage, costs, g, logits, ranges, labels, tl, ul, 0))
    assert np.array_equal(fin, ul + 1 <= R)


@pytest.mark.parametrize("storage", ["fp32", "fp64", "bf16"])
def test_no_labels(wr, storage):
    """U = 1: windows starting at -1 or 0 both cover u = 0; only blanks, every utterance has its path."""
    N, T, U, V, R = 4, 8, 1, 1030, 2
    rng, logits, labels, tl, ul = make("U1", storage, N, T, U, V, R, 0)
    ranges = -rng.integers(0, 2, size=(N, T)).astype(np.int32)
    costs, g, _, _ = run(wr, storage, logits, ranges, labels, tl, ul, U, 0, lam=0.5)
    assert np.isfinite(check(storage, costs, g, logits, ranges, labels, tl, ul, 0, lam=0.5)).all()


# ---- misaligned logits ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V,offset,family,a,b", [
    (50, 1, "tile", 1, 8),      # aligned: chunk kernels
    (100, 1, "tile", 1, 16),    # aligned: chunk kernels
    (100, 2, "tile", 2, 8),     # 8-byte aligned: float2
    (5000, 1, "row", 1, 8),     # aligned: grad_row_kernel<float, 4, 5>
    (5000, 2, "row", 2, 8),
])
def test_misaligned_logits(wr, V, offset, family, a, b):
    """Logits and gradient as contiguous views `offset` fp32 elements into larger buffers leave the chunk kernels and
    the 16-byte vectors; the result matches the aligned call within the fp32 tolerance, and the reference."""
    N, T, U, R = 3, 7, 5, 3
    name = "misaligned_V%d" % V
    rng, logits, labels, tl, ul = make(name, "fp32", N, T, U, V, R, 0)
    ranges = windows(rng, tl, ul, T, R)
    c0, g0, _, _ = run(wr, "fp32", logits, ranges, labels, tl, ul, U, 0, lam=0.5)
    c1, g1, kernels, _ = run(wr, "fp32", logits, ranges, labels, tl, ul, U, 0, lam=0.5, offset=offset)
    assert_launched(kernels, *heads("fp32", family, a, b, reg=True))
    fin = np.isfinite(c0)
    assert np.array_equal(fin, np.isfinite(c1)) and np.allclose(c1[fin], c0[fin], rtol=1e-5, atol=0)
    assert (np.abs(g1 - g0) <= 1e-4 * np.abs(g0) + 1e-6).all(), np.abs(g1 - g0).max()
    check("fp32", c1, g1, logits, ranges, labels, tl, ul, 0, lam=0.5)


# ---- grouped schedule -----------------------------------------------------------------------------------------------
def test_grouped_schedule_matches_the_split_backward(wr):
    """N = 16, T = 1500, U = 301, R = 8, V = 600 (fp32, 461 MB of logits).  The streaming passes' estimate,
    192000 rows x 600 x 12 B / 3 TB/s = 461 us, is past 400 us, and the lattice's, 0.25 us x 1801 + 20 = 470 us, is
    past 8 % of it.  So the full call runs 4 batch groups (offset by maxT * R rows) behind one fill of the whole
    lattice: 13 launches, each group's multi-warp lattice with a ring of 16 diagonals.  The split forward + backward
    never groups; the per-row arithmetic is the same, so both agree bit for bit.  Two utterances, in the first and
    the last group, against the reference."""
    N, T, U, V, R, blank = 16, 1500, 301, 600, 8, 0
    lam, clamp = 0.01, 0.05
    rng = np.random.default_rng(71)
    labels = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    tl = rng.integers(T // 2, T + 1, size=N).astype(np.int32)
    ul = rng.integers(U // 2, U, size=N).astype(np.int32)
    tl[0], ul[0] = T, U - 1
    ranges = windows(rng, tl, ul, T, R)
    gen = torch.Generator("cuda").manual_seed(71)
    x = torch.randn(N, T, R, V, device="cuda", generator=gen) * 2
    rg, lab, tld, uld = (torch.as_tensor(a).cuda() for a in (ranges, labels, tl, ul))
    from warprnnt_pytorch.pruned import pruned_workspace_size
    opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream().cuda_stream, blank_label=blank,
                         maxT=T, maxU=U, batch_first=True)
    gopt = wr.rnntGradOptions(lam, clamp)
    ws = torch.empty(pruned_workspace_size(T, U, R, N, 4), dtype=torch.uint8, device="cuda")
    lib = wr.lib()

    c_full = torch.empty(N, device="cuda")
    g_full = torch.empty_like(x)

    def call():
        c_full.fill_(float("nan"))
        g_full.fill_(float("nan"))
        st = lib.rnnt_b200_pruned_loss_async_ex(0, 0, x.data_ptr(), g_full.data_ptr(), rg.data_ptr(), R,
                                                lab.data_ptr(), uld.data_ptr(), tld.data_ptr(), V, N,
                                                c_full.data_ptr(), 1.0, gopt, ws.data_ptr(), opt)
        assert st == 0, wr.status_string(st)
        return wr.last_launch_count()

    launches, kernels = profiled(call)
    assert launches == 13   # the fill, then 4 x (pass 1, lattice, pass 2)
    # next to other groups' streaming passes a lattice keeps 16 diagonals in flight, not 8 (lattice_ring_depth)
    assert_launched(kernels, *heads("fp32", "tile", 4, 32, reg=True), "lattice_lin_kernel<1, true, 16>")

    c_split = torch.full((N,), float("nan"), device="cuda")
    g_split = torch.full_like(x, float("nan"))
    st = lib.rnnt_b200_pruned_forward(0, x.data_ptr(), rg.data_ptr(), R, lab.data_ptr(), uld.data_ptr(),
                                      tld.data_ptr(), V, N, c_split.data_ptr(), 1, ws.data_ptr(), opt)
    assert st == 0, wr.status_string(st)
    st = lib.rnnt_b200_pruned_backward_ex(0, x.data_ptr(), g_split.data_ptr(), rg.data_ptr(), R, lab.data_ptr(),
                                          uld.data_ptr(), tld.data_ptr(), V, N, None, 1.0, gopt, ws.data_ptr(), opt)
    assert st == 0, wr.status_string(st)
    torch.cuda.synchronize()
    assert torch.equal(c_split, c_full) and torch.equal(g_split, g_full)
    del g_split

    c = c_full.double().cpu().numpy()
    assert np.isinf(c[N - 1]) and np.isfinite(c[0])
    for b in (0, 13):
        Tb = int(tl[b])
        logits = x[b:b + 1, :Tb].double().cpu().numpy()
        g = g_full[b:b + 1, :Tb].double().cpu().numpy()
        check("fp32", c[b:b + 1], g, logits, ranges[b:b + 1, :Tb], labels[b:b + 1], tl[b:b + 1], ul[b:b + 1], blank,
              lam, clamp)
        assert not g_full[b, Tb:].any()
