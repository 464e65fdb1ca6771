"""Argument rules of the fused joiner's C-ABI (rnnt_b200_joiner_workspace_size / _forward / _backward) and of the
Python functions, and the workspace's memory contract, without a GPU.

Every call is rejected by the host-side checks before any device access (the buffers are host memory).  Status 2 is
RNNT_STATUS_INVALID_VALUE; 3 is what the CPU location returns, so a call that returns 3 passed every argument
check."""
import ctypes as C

import pytest
import torch

FWD = "act enc pred w bias labels ylen xlen H V N chunk px py ws opt".split()
BWD = "act enc pred w bias labels ylen xlen H V N chunk dpx dpy ge gp gw gb ws opt".split()
POINTERS = {"enc", "pred", "w", "bias", "labels", "ylen", "xlen", "px", "py", "ws", "dpx", "dpy", "ge", "gp", "gw",
            "gb"}
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
        vals = dict(act=0, H=16, V=5, N=2, chunk=0)
        vals.update({p: self.addr for p in POINTERS})
        vals.update(kw)
        opt = self.wr.rnntOptions()
        opt.loc, opt.maxT, opt.maxU, opt.blank_label = loc, maxT, maxU, blank
        vals["opt"] = opt
        return self.fn(*[vals[p] for p in self.params])


@pytest.fixture(params=["rnnt_b200_joiner_forward", "rnnt_b200_joiner_backward"], scope="module")
def entry(request, wr, jn, buf):
    return Caller(wr, jn, request.param, FWD if request.param.endswith("forward") else BWD, buf)


def test_valid_arguments_reach_the_location_check(entry):
    for act in (0, 1):
        assert entry(loc=0, act=act) == 3
    assert entry(loc=0, maxT=1, maxU=1) == 3
    assert entry(loc=0, maxU=1024) == 3
    assert entry(loc=0, H=1024, V=2, blank=1) == 3
    assert entry(loc=0, chunk=1) == 3
    assert entry(loc=0, V=5001, blank=5000) == 3
    for q in OPTIONAL & set(entry.params):
        assert entry(loc=0, **{q: None}) == 3
    for q in NO_LABELS & set(entry.params):
        assert entry(loc=0, maxU=1, **{q: None}) == 3


def test_extents_and_options(entry):
    bad = [dict(act=-1), dict(act=2), dict(H=0), dict(H=8), dict(H=24), dict(H=1040), dict(V=1), dict(V=0),
           dict(blank=-1), dict(blank=5), dict(chunk=-1), dict(N=0), dict(maxT=0), dict(maxU=0), dict(maxU=1025),
           dict(N=1 << 12, maxT=1 << 10, maxU=1 << 9)]
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
    f = jn._lib.rnnt_b200_joiner_workspace_size
    assert f(4, 3, 2, 16, 5, 0, C.byref(n)) == 0 and n.value > 0
    for args in [(0, 3, 2, 16, 5, 0), (4, 0, 2, 16, 5, 0), (4, 3, 0, 16, 5, 0), (4, 1025, 2, 16, 5, 0),
                 (4, 3, 2, 8, 5, 0), (4, 3, 2, 1040, 5, 0), (4, 3, 2, 16, 1, 0), (4, 3, 2, 16, 5, -1),
                 (1 << 10, 1 << 9, 1 << 12, 16, 5, 0)]:
        assert f(*args, C.byref(n)) == 2, args
    assert f(4, 3, 2, 16, 5, 0, None) == 2


def _scratch_bound(T, U, N, H, V):
    """Bytes of everything but the chunk scratch: lse per cell and the fp32 accumulators (dW in at most 16 slabs)."""
    Hp, Vp = (H + 64) // 64 * 64, (V + 63) // 64 * 64
    return N * T * U * 4 + N * T * H * 4 + N * U * H * 4 + 16 * Vp * Hp * 4 + 4 * 256


@pytest.mark.parametrize("V", [5000, 50000])
def test_default_scratch_is_at_most_256_mib(jn, V):
    T, U, N, H = 150, 21, 128, 640
    size = jn.workspace_size(T, U, N, H, V)
    Hp, Vp = (H + 64) // 64 * 64, (V + 63) // 64 * 64
    fixed = N * T * U * 4 + N * T * H * 4 + N * U * H * 4 + Vp * Hp * 4     # one dW slab at these widths
    assert size - fixed <= (256 << 20) + 4 * 256
    assert size < N * T * U * V * 2 / 8           # far below the bf16 logits alone


def test_workspace_does_not_grow_with_the_alphabet_beyond_the_scratch(jn):
    T, U, N, H = 50, 11, 8, 256
    for chunk in (64, 1000):
        for V in (2, 500, 5000, 50000):
            size = jn.workspace_size(T, U, N, H, V, chunk)
            rows = (chunk + 127) // 128 * 128
            Hp, Vp = (H + 64) // 64 * 64, (V + 63) // 64 * 64
            assert size <= _scratch_bound(T, U, N, H, V) + rows * (Hp * 2 + Vp * 2 + H * 4), (chunk, V)
            assert size < N * T * U * V * 4 or V == 2


def test_chunk_is_capped_at_the_cell_count(jn):
    assert jn.workspace_size(4, 3, 2, 16, 5, 10 ** 6) == jn.workspace_size(4, 3, 2, 16, 5, 24)
    assert jn.workspace_size(4, 3, 2, 16, 5) == jn.workspace_size(4, 3, 2, 16, 5, 24)


def _args(N=2, T=4, U=3, H=16, V=5, dtype=torch.bfloat16):
    return dict(enc=torch.zeros(N, T, H, dtype=dtype), pred=torch.zeros(N, U, H, dtype=dtype),
                weight=torch.zeros(V, H, dtype=dtype), bias=torch.zeros(V, dtype=dtype),
                labels=torch.zeros(N, U - 1, dtype=torch.int32), act_lens=torch.full((N,), T, dtype=torch.int32),
                label_lens=torch.full((N,), U - 1, dtype=torch.int32))


def _call(f, a, **kw):
    return f(a["enc"], a["pred"], a["weight"], a["bias"], a["labels"], a["act_lens"], a["label_lens"], **kw)


@pytest.mark.parametrize("fn", ["joiner_log_probs", "joiner_rnnt_loss"])
def test_python_argument_errors(fn):
    import warprnnt_pytorch as w
    f = getattr(w, fn)
    with pytest.raises(RuntimeError, match="CUDA"):
        _call(f, _args())
    for dtype in (torch.float16, torch.float32):
        with pytest.raises(TypeError):
            _call(f, _args(dtype=dtype))
        a = _args()
        a["weight"] = a["weight"].to(dtype)
        with pytest.raises(TypeError):
            _call(f, a)
    for key, dtype in (("labels", torch.int64), ("act_lens", torch.int64), ("label_lens", torch.float32)):
        a = _args()
        a[key] = a[key].to(dtype)
        with pytest.raises(TypeError):
            _call(f, a)
    bad = [dict(H=8), dict(H=24), dict(H=1040), dict(V=1), dict(U=1025, T=1, N=1)]
    for kw in bad:
        with pytest.raises(ValueError):
            _call(f, _args(**kw))
    for mutate in (lambda a: a.update(enc=a["enc"].transpose(0, 1).contiguous().transpose(0, 1)),
                   lambda a: a.update(pred=a["pred"][:, :2]),
                   lambda a: a.update(weight=a["weight"][:, :8].contiguous()),
                   lambda a: a.update(bias=a["bias"][:3]),
                   lambda a: a.update(labels=a["labels"][:, :1].contiguous()),
                   lambda a: a.update(act_lens=a["act_lens"][:1]),
                   lambda a: a.update(label_lens=a["label_lens"][:1]),
                   lambda a: a.update(enc=a["enc"][0])):
        a = _args()
        mutate(a)
        with pytest.raises(ValueError):
            _call(f, a)
    for kw in (dict(blank=5), dict(blank=-1), dict(activation='gelu')):
        with pytest.raises(ValueError):
            _call(f, _args(), **kw)
    if fn == "joiner_log_probs":
        for chunk in (0, -1, 1.5, True):
            with pytest.raises(ValueError):
                _call(f, _args(), chunk_cells=chunk)
    else:
        for kw in (dict(reduction='avg'), dict(rnnt_type='constrained'), dict(delay_penalty=-1.0)):
            with pytest.raises(ValueError):
                _call(f, _args(), **kw)


def test_module_rejects_bad_options():
    import warprnnt_pytorch as w
    for kw in (dict(reduction='avg'), dict(activation='gelu'), dict(rnnt_type='constrained'),
               dict(delay_penalty=float('nan'))):
        with pytest.raises(ValueError):
            w.JoinerRNNTLoss(**kw)
