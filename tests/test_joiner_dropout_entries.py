"""Argument rules of the dropout entries of the fused and pruned fused joiners (rnnt_b200_joiner_forward_drop /
_backward_drop, rnnt_b200_pruned_joiner_forward_drop / _backward_drop) and of the Python functions' and modules'
dropout arguments, without a GPU.

Every call is rejected by the host-side checks before any device access (the buffers are host memory).  Status 2 is
RNNT_STATUS_INVALID_VALUE; 3 is what the CPU location returns, so a call that returns 3 passed every argument
check."""
import ctypes as C

import pytest
import torch

DENSE_FWD = "act enc pred w bias labels ylen xlen H V N chunk px py drop ws opt".split()
DENSE_BWD = "act enc pred w bias labels ylen xlen H V N chunk dpx dpy ge gp gw gb drop ws opt".split()
PRUNED_FWD = "act enc pred w bias labels ylen xlen ranges R H V N chunk px py drop ws opt".split()
PRUNED_BWD = "act enc pred w bias labels ylen xlen ranges R H V N chunk dpx dpy ge gp gw gb drop ws opt".split()
ENTRIES = {"rnnt_b200_joiner_forward_drop": DENSE_FWD, "rnnt_b200_joiner_backward_drop": DENSE_BWD,
           "rnnt_b200_pruned_joiner_forward_drop": PRUNED_FWD, "rnnt_b200_pruned_joiner_backward_drop": PRUNED_BWD}
POINTERS = {"enc", "pred", "w", "bias", "labels", "ylen", "xlen", "ranges", "px", "py", "ws", "dpx", "dpy", "ge",
            "gp", "gw", "gb"}
OPTIONAL = {"bias", "gb"}


@pytest.fixture(scope="module")
def jn():
    import warprnnt_pytorch.joiner as jn
    return jn


@pytest.fixture(scope="module")
def buf():
    return (C.c_byte * 4096)()     # 16-byte aligned host memory standing in for every device buffer


class Caller:
    def __init__(self, jn, name, params, buf):
        self.jn, self.fn, self.params = jn, getattr(jn._lib, name), params
        self.addr = C.addressof(buf)
        self.addr += (-self.addr) % 16

    def __call__(self, loc=1, maxT=4, maxU=3, blank=0, p=0.2, seed="ok", **kw):
        import warprnnt_pytorch.warp_rnnt as wr
        vals = dict(act=0, H=16, V=5, N=2, chunk=0, R=2)
        vals.update({q: self.addr for q in POINTERS})
        vals["drop"] = self.jn.rnntJoinerDropout(p, self.addr + 64 if seed == "ok" else seed)
        vals.update(kw)
        opt = wr.rnntOptions()
        opt.loc, opt.maxT, opt.maxU, opt.blank_label = loc, maxT, maxU, blank
        vals["opt"] = opt
        return self.fn(*[vals[q] for q in self.params])


@pytest.fixture(params=sorted(ENTRIES), scope="module")
def entry(request, jn, buf):
    return Caller(jn, request.param, ENTRIES[request.param], buf)


def test_valid_dropout_reaches_the_location_check(entry):
    for p in (0.0, 1e-9, 0.1, 0.2, 0.5, 0.999, 1 - 2 ** -24):   # 1 - 2^-24: the largest float32 below 1
        for act in (0, 1):
            assert entry(loc=0, p=p, act=act) == 3, p
    assert entry(loc=0, p=0.0, seed=None) == 3            # no seed is needed without dropout
    assert entry(loc=0, p=0.0, seed=entry.addr + 8) == 3  # 8-byte alignment is enough
    assert entry(loc=0, p=0.2, seed=entry.addr + 8) == 3
    assert entry(loc=0, p=0.2, maxT=1, maxU=1, R=1, labels=None) == 3


def test_dropout_rules(entry):
    bad = [dict(p=float("nan")), dict(p=-0.1), dict(p=-1e-40), dict(p=1.0), dict(p=1.5), dict(p=float("inf")),
           dict(p=-float("inf")), dict(p=0.2, seed=None), dict(p=1e-9, seed=None), dict(seed=entry.addr + 4),
           dict(p=0.0, seed=entry.addr + 4), dict(p=0.5, seed=entry.addr + 1)]
    for kw in bad:
        assert entry(**kw) == 2, kw
        assert entry(loc=0, **kw) == 2, kw


def test_every_plain_rule_still_applies(entry):
    bad = [dict(act=2), dict(H=24), dict(V=1), dict(blank=5), dict(chunk=-1), dict(maxU=1025)]
    if "R" in entry.params:
        bad += [dict(R=0), dict(ranges=None)]
    for kw in bad:
        assert entry(**kw) == 2, kw
        assert entry(loc=0, **kw) == 2, kw
    for q in POINTERS & set(entry.params):
        if q not in OPTIONAL:
            assert entry(**{q: None}) == 2, q
        if q in {"enc", "pred", "w", "ws"}:
            assert entry(**{q: entry.addr + 8}) == 2, q


def _plain_size(T, U, N, H, V, chunk, rows_per_frame):
    """The plain calls' workspace for an explicit chunk: per-row lse, the fp32 accumulators of d_enc, d_pred and the
    dW slabs, and the h, dlogits and ds scratch, each 256-byte aligned.  Nothing for a mask."""
    up = lambda x, a: -(-x // a) * a
    Hp, Vp = up(H + 1, 64), up(V, 64)
    cells = N * T * rows_per_frame
    rows = up(min(chunk, cells), 128)
    slabs = min(-(-264 // ((Vp // 64) * (Hp // 64))), 16, rows // 64)
    o = 0
    for n in (cells * 4, N * T * H * 4, N * U * H * 4, slabs * Vp * Hp * 4, rows * Hp * 2, rows * Vp * 2,
              rows * H * 4):
        o = up(o + n, 256)
    return o


def test_workspace_sizes_are_the_plain_calls(jn):
    """The dropout calls run in the workspace the plain workspace-size entries report: the mask is regenerated,
    never stored, and the ds epilogue recomputes tanh's h instead of keeping a second copy."""
    T, U, N, H, V = 50, 11, 8, 256, 500
    for chunk in (64, 1000, 4400):
        assert jn.workspace_size(T, U, N, H, V, chunk) == _plain_size(T, U, N, H, V, chunk, U)
        for R in (2, 5):
            assert jn.workspace_size(T, U, N, H, V, chunk, s_range=R) == _plain_size(T, U, N, H, V, chunk, R)


def _args(N=2, T=4, U=3, H=16, V=5, dtype=torch.bfloat16):
    return dict(enc=torch.zeros(N, T, H, dtype=dtype), pred=torch.zeros(N, U, H, dtype=dtype),
                weight=torch.zeros(V, H, dtype=dtype), bias=torch.zeros(V, dtype=dtype),
                labels=torch.zeros(N, U - 1, dtype=torch.int32), act_lens=torch.full((N,), T, dtype=torch.int32),
                label_lens=torch.full((N,), U - 1, dtype=torch.int32), ranges=torch.zeros(N, T, dtype=torch.int32))


FUNCTIONS = ["joiner_log_probs", "joiner_rnnt_loss", "JoinerRNNTLoss", "pruned_joiner_log_probs",
             "pruned_joiner_rnnt_loss", "PrunedJoinerRNNTLoss"]


def _call(fn, a, **kw):
    import warprnnt_pytorch as w
    head = (a["enc"], a["pred"], a["weight"], a["bias"], a["labels"], a["act_lens"], a["label_lens"])
    window = (a["ranges"], 2) if fn.startswith(("pruned", "Pruned")) else ()
    if fn[0].isupper():
        return getattr(w, fn)(dropout=kw.pop("dropout", 0.2))(*head, *window)
    return getattr(w, fn)(*head, *window, **kw)


BAD_P = [float("nan"), -0.1, 1.0, 1.5, float("inf"), True, False, "0.2", None, 1 - 2 ** -30]


@pytest.mark.parametrize("fn", FUNCTIONS)
def test_python_dropout_errors(fn):
    for p in BAD_P:
        with pytest.raises(ValueError, match="dropout"):
            _call(fn, _args(), dropout=p)
    with pytest.raises(RuntimeError, match="CUDA"):   # a valid p reaches the device check of the inputs
        _call(fn, _args(), dropout=0.2)


@pytest.mark.parametrize("fn", [f for f in FUNCTIONS if f[0].islower()])
def test_python_seed_errors(fn):
    for seed in (torch.zeros(1, dtype=torch.int32), torch.zeros(1, dtype=torch.float64),
                 torch.zeros(1, dtype=torch.uint8), 7, 2.0, [1]):
        with pytest.raises(TypeError, match="dropout_seed"):
            _call(fn, _args(), dropout=0.2, dropout_seed=seed)
    for seed in (torch.zeros(2, dtype=torch.int64), torch.zeros(0, dtype=torch.int64),
                 torch.zeros(1, 2, dtype=torch.int64)):
        with pytest.raises(ValueError, match="dropout_seed"):
            _call(fn, _args(), dropout=0.2, dropout_seed=seed)
    for shape in ((), (1,), (1, 1)):   # one element of any shape passes, and a CPU tensor is a RuntimeError
        with pytest.raises(RuntimeError):
            _call(fn, _args(), dropout=0.2, dropout_seed=torch.zeros(shape, dtype=torch.int64))


def test_seed_on_another_device_is_a_runtime_error(jn):
    """The device rule of an explicit seed, checked on its own (the inputs' device check runs first)."""
    with pytest.raises(RuntimeError, match="device"):
        jn._seed_on(torch.zeros(1, dtype=torch.int64), torch.device("cuda", 0))


def test_dropout_p_accepts_what_the_abi_takes(jn):
    assert jn.dropout_p(0) == 0.0 and jn.dropout_p(0.2) == 0.2 and jn.dropout_p(0.5) == 0.5
    assert jn.dropout_p(1 - 2 ** -20) == 1 - 2 ** -20
    for p in BAD_P:
        with pytest.raises(ValueError):
            jn.dropout_p(p)


def test_modules_keep_their_dropout_and_reject_bad_ones():
    import warprnnt_pytorch as w
    for cls in (w.JoinerRNNTLoss, w.PrunedJoinerRNNTLoss):
        assert cls().dropout == 0.0
        assert cls(activation='relu', dropout=0.2).dropout == 0.2
        for p in BAD_P:
            with pytest.raises(ValueError):
                cls(dropout=p)


def test_low_level_dropout_calls_need_their_seed(jn):
    """gpu_joiner_forward / _backward with dropout > 0 and no seed tensor are rejected before any device work."""
    a = _args()
    px, py = torch.zeros(2, 2, 4), torch.zeros(2, 3, 4)
    head = (a["enc"], a["pred"], a["weight"], a["bias"], a["labels"], a["act_lens"], a["label_lens"])
    g = [torch.zeros_like(a[k]) for k in ("enc", "pred", "weight", "bias")]
    ws = torch.zeros(jn.workspace_size(4, 3, 2, 16, 5), dtype=torch.uint8)
    with pytest.raises(ValueError, match="seed"):
        jn.gpu_joiner_forward(*head, px, py, 0, "tanh", None, ws, dropout=0.2)
    with pytest.raises(ValueError, match="seed"):
        jn.gpu_joiner_backward(*head, px, py, *g, 0, "tanh", None, ws, dropout=0.2)
