"""Argument rules of the pruned fused joiner's C-ABI (rnnt_b200_pruned_joiner_workspace_size / _forward / _backward)
and of the Python functions, and the workspace's memory contract, without a GPU.

Every call is rejected by the host-side checks before any device access (the buffers are host memory).  Status 2 is
RNNT_STATUS_INVALID_VALUE; 3 is what the CPU location returns, so a call that returns 3 passed every argument
check."""
import ctypes as C

import pytest
import torch

FWD = "act enc pred w bias labels ylen xlen ranges R H V N chunk px py ws opt".split()
BWD = "act enc pred w bias labels ylen xlen ranges R H V N chunk dpx dpy ge gp gw gb ws opt".split()
POINTERS = {"enc", "pred", "w", "bias", "labels", "ylen", "xlen", "ranges", "px", "py", "ws", "dpx", "dpy", "ge",
            "gp", "gw", "gb"}
OPTIONAL = {"bias", "gb"}
NO_LABELS = {"labels", "px", "dpx"}          # may be NULL when maxU == 1


@pytest.fixture(scope="module")
def wr():
    import warprnnt_pytorch.warp_rnnt as wr
    return wr


@pytest.fixture(scope="module")
def jn():
    import warprnnt_pytorch.joiner as jn
    return jn


@pytest.fixture(scope="module")
def buf():
    return (C.c_byte * 4096)()     # 16-byte aligned host memory standing in for every device buffer


class Caller:
    def __init__(self, wr, jn, name, params, buf):
        self.wr, self.fn, self.params = wr, getattr(jn._lib, name), params
        self.addr = C.addressof(buf)
        self.addr += (-self.addr) % 16

    def __call__(self, loc=1, maxT=4, maxU=3, blank=0, **kw):
        vals = dict(act=0, H=16, V=5, N=2, chunk=0, R=2)
        vals.update({p: self.addr for p in POINTERS})
        vals.update(kw)
        opt = self.wr.rnntOptions()
        opt.loc, opt.maxT, opt.maxU, opt.blank_label = loc, maxT, maxU, blank
        vals["opt"] = opt
        return self.fn(*[vals[p] for p in self.params])


@pytest.fixture(params=["rnnt_b200_pruned_joiner_forward", "rnnt_b200_pruned_joiner_backward"], scope="module")
def entry(request, wr, jn, buf):
    return Caller(wr, jn, request.param, FWD if request.param.endswith("forward") else BWD, buf)


def test_valid_arguments_reach_the_location_check(entry):
    for act in (0, 1):
        assert entry(loc=0, act=act) == 3
    assert entry(loc=0, maxT=1, maxU=1, R=1) == 3
    assert entry(loc=0, maxU=1024, R=1024) == 3
    assert entry(loc=0, R=5000) == 3                     # R > U is allowed
    assert entry(loc=0, H=1024, V=2, blank=1) == 3
    assert entry(loc=0, chunk=1) == 3
    assert entry(loc=0, V=5001, blank=5000) == 3
    assert entry(loc=0, N=1 << 10, maxT=1 << 10, maxU=2, R=(1 << 11) - 1) == 3   # N T R just below 2^31
    for q in OPTIONAL & set(entry.params):
        assert entry(loc=0, **{q: None}) == 3
    for q in NO_LABELS & set(entry.params):
        assert entry(loc=0, maxU=1, **{q: None}) == 3


def test_window_rules(entry):
    bad = [dict(R=0), dict(R=-1), dict(R=-(1 << 31)), dict(ranges=None), dict(N=1 << 10, maxT=1 << 10, R=1 << 11),
           dict(N=1 << 12, maxT=1 << 10, maxU=2, R=1 << 9)]
    for kw in bad:
        assert entry(**kw) == 2, kw
        assert entry(loc=0, **kw) == 2, kw


def test_extents_and_options(entry):
    bad = [dict(act=-1), dict(act=2), dict(H=0), dict(H=8), dict(H=24), dict(H=1040), dict(V=1), dict(V=0),
           dict(blank=-1), dict(blank=5), dict(chunk=-1), dict(N=0), dict(maxT=0), dict(maxU=0), dict(maxU=1025),
           dict(N=1 << 12, maxT=1 << 10, maxU=1 << 9, R=1)]
    for kw in bad:
        assert entry(**kw) == 2, kw
        assert entry(loc=0, **kw) == 2, kw


def test_null_and_misaligned_pointers(entry):
    for q in POINTERS & set(entry.params):
        if q not in OPTIONAL:
            assert entry(**{q: None}) == 2, q
            assert entry(loc=0, **{q: None}) == 2, q
        if q in {"enc", "pred", "w", "ws"}:
            assert entry(**{q: entry.addr + 8}) == 2, q
    assert entry(bias=entry.addr + 1) == 2


def test_workspace_size_rules(jn):
    n = C.c_size_t(0)
    f = jn._lib.rnnt_b200_pruned_joiner_workspace_size
    assert f(4, 3, 2, 2, 16, 5, 0, C.byref(n)) == 0 and n.value > 0
    assert f(4, 3, 9, 2, 16, 5, 0, C.byref(n)) == 0                      # R > U
    for args in [(0, 3, 2, 2, 16, 5, 0), (4, 0, 2, 2, 16, 5, 0), (4, 3, 2, 0, 16, 5, 0), (4, 1025, 2, 2, 16, 5, 0),
                 (4, 3, 2, 2, 8, 5, 0), (4, 3, 2, 2, 1040, 5, 0), (4, 3, 2, 2, 16, 1, 0), (4, 3, 2, 2, 16, 5, -1),
                 (4, 3, 0, 2, 16, 5, 0), (4, 3, -3, 2, 16, 5, 0), (1 << 10, 2, 1 << 11, 1 << 10, 16, 5, 0),
                 (1 << 10, 1 << 9, 1, 1 << 12, 16, 5, 0)]:
        assert f(*args, C.byref(n)) == 2, args
    assert f(4, 3, 2, 2, 16, 5, 0, None) == 2


def _fixed(T, U, R, N, H, V, slabs=16):
    """Bytes of everything but the chunk scratch: lse per row and the fp32 accumulators (dW in at most 16 slabs)."""
    Hp, Vp = (H + 64) // 64 * 64, (V + 63) // 64 * 64
    return N * T * R * 4 + N * T * H * 4 + N * U * H * 4 + slabs * Vp * Hp * 4 + 4 * 256


def test_lse_grows_with_the_rows_and_nothing_with_the_alphabet_times_the_cells(jn):
    T, U, N, H = 50, 11, 8, 256
    for chunk in (64, 1000):
        for V in (2, 500, 5000, 50000):
            sizes = [jn.workspace_size(T, U, N, H, V, chunk, s_range=R) for R in (1, 2, 5, 11, 40)]
            for R, size in zip((1, 2, 5, 11, 40), sizes):
                rows = (min(chunk, N * T * R) + 127) // 128 * 128
                Hp, Vp = (H + 64) // 64 * 64, (V + 63) // 64 * 64
                assert size <= _fixed(T, U, R, N, H, V) + rows * (Hp * 2 + Vp * 2 + H * 4), (chunk, V, R)
                # twice the utterances, once the chunk is full: the per-row lse and the d_enc / d_pred
                # accumulators grow, nothing of width V does
                if chunk <= N * T * R:
                    grow = jn.workspace_size(T, U, 2 * N, H, V, chunk, s_range=R) - size
                    assert grow <= N * T * R * 4 + N * T * H * 4 + N * U * H * 4 + 3 * 256, (chunk, V, R)
            # the per-row lse: 4 N T bytes more per window row (the scratch is fixed once the chunk fits)
            assert sizes[-1] - sizes[-2] >= 4 * N * T * (40 - 11) - 256
            assert sizes[-1] - sizes[-2] <= 4 * N * T * (40 - 11) + 2 * 256


def test_window_of_the_whole_lattice_sizes_as_the_dense_joiner(jn):
    for chunk in (None, 64, 1000):
        assert jn.workspace_size(9, 5, 4, 64, 300, chunk, s_range=5) == jn.workspace_size(9, 5, 4, 64, 300, chunk)


@pytest.mark.parametrize("V", [5000, 32000])
def test_default_scratch_is_at_most_256_mib(jn, V):
    T, U, N, H, R = 500, 101, 64, 640, 5
    size = jn.workspace_size(T, U, N, H, V, s_range=R)
    Hp, Vp = (H + 64) // 64 * 64, (V + 63) // 64 * 64
    slabs = min(-(-264 // ((Vp // 64) * (Hp // 64))), 16)
    assert size - _fixed(T, U, R, N, H, V, slabs) <= (256 << 20)
    assert size < N * T * R * V * 2 / 4           # a fraction of the bf16 pruned logits alone


def _args(N=2, T=4, U=3, H=16, V=5, dtype=torch.bfloat16):
    return dict(enc=torch.zeros(N, T, H, dtype=dtype), pred=torch.zeros(N, U, H, dtype=dtype),
                weight=torch.zeros(V, H, dtype=dtype), bias=torch.zeros(V, dtype=dtype),
                labels=torch.zeros(N, U - 1, dtype=torch.int32), act_lens=torch.full((N,), T, dtype=torch.int32),
                label_lens=torch.full((N,), U - 1, dtype=torch.int32), ranges=torch.zeros(N, T, dtype=torch.int32))


def _call(f, a, s_range=2, **kw):
    return f(a["enc"], a["pred"], a["weight"], a["bias"], a["labels"], a["act_lens"], a["label_lens"], a["ranges"],
             s_range, **kw)


@pytest.mark.parametrize("fn", ["pruned_joiner_log_probs", "pruned_joiner_rnnt_loss", "PrunedJoinerRNNTLoss"])
def test_python_argument_errors(fn):
    import warprnnt_pytorch as w
    if fn == "PrunedJoinerRNNTLoss":
        f = w.PrunedJoinerRNNTLoss()
    else:
        f = getattr(w, fn)
    with pytest.raises(RuntimeError, match="CUDA"):
        _call(f, _args())
    for dtype in (torch.float16, torch.float32):
        with pytest.raises(TypeError):
            _call(f, _args(dtype=dtype))
    for key, dtype in (("labels", torch.int64), ("act_lens", torch.int64), ("ranges", torch.int64),
                       ("ranges", torch.float32)):
        a = _args()
        a[key] = a[key].to(dtype)
        with pytest.raises(TypeError):
            _call(f, a)
    for s_range in (0, -1, 2.0, True, None):
        with pytest.raises(ValueError):
            _call(f, _args(), s_range=s_range)
    for s_range in (2, 5, None):   # a missing window is an error, never the dense joiner
        a = _args()
        a["ranges"] = None
        with pytest.raises(TypeError, match="ranges"):
            _call(f, a, s_range=s_range)
    with pytest.raises(ValueError):
        _call(f, _args(N=1 << 10, T=1 << 10, H=16), s_range=1 << 11)    # N T R = 2^31
    for mutate in (lambda a: a.update(ranges=a["ranges"][:, :3]),
                   lambda a: a.update(ranges=a["ranges"][:1]),
                   lambda a: a.update(ranges=a["ranges"][0]),
                   lambda a: a.update(ranges=a["ranges"][:, None, :]),
                   lambda a: a.update(ranges=torch.zeros(4, 2, dtype=torch.int32).t()),
                   lambda a: a.update(pred=a["pred"][:, :2]),
                   lambda a: a.update(enc=a["enc"][0])):
        a = _args()
        mutate(a)
        with pytest.raises(ValueError):
            _call(f, a)
    bad = [dict(H=8), dict(V=1), dict(U=1025, T=1, N=1)]
    for kw in bad:
        with pytest.raises(ValueError):
            _call(f, _args(**kw))
    if fn == "pruned_joiner_log_probs":
        for kw in (dict(blank=5), dict(activation='gelu'), dict(chunk_cells=0)):
            with pytest.raises(ValueError):
                _call(f, _args(), **kw)
    elif fn == "pruned_joiner_rnnt_loss":
        for kw in (dict(reduction='avg'), dict(rnnt_type='constrained'), dict(delay_penalty=-1.0), dict(blank=-1)):
            with pytest.raises(ValueError):
                _call(f, _args(), **kw)


def test_module_rejects_bad_options():
    import warprnnt_pytorch as w
    for kw in (dict(reduction='avg'), dict(activation='gelu'), dict(rnnt_type='constrained'),
               dict(delay_penalty=float('nan'))):
        with pytest.raises(ValueError):
            w.PrunedJoinerRNNTLoss(**kw)


def test_low_level_calls_need_the_whole_window(jn):
    """gpu_joiner_forward / _backward: ranges or s_range alone is rejected before any device work."""
    a = _args()
    px, py = torch.zeros(2, 2, 4), torch.zeros(2, 3, 4)
    head = (a["enc"], a["pred"], a["weight"], a["bias"], a["labels"], a["act_lens"], a["label_lens"])
    g = [torch.zeros_like(a[k]) for k in ("enc", "pred", "weight", "bias")]
    for window in (dict(ranges=a["ranges"]), dict(s_range=2), dict(ranges=None, s_range=5)):
        with pytest.raises(ValueError, match="both ranges and s_range"):
            jn.gpu_joiner_forward(*head, px, py, 0, "tanh", **window)
        with pytest.raises(ValueError, match="both ranges and s_range"):
            jn.gpu_joiner_backward(*head, px, py, *g, 0, "tanh", None, torch.zeros(16, dtype=torch.uint8), **window)
