"""Argument rules of the lattice-option (delay penalty) entries of the C-ABI and of the Python keyword, without a GPU.

As in test_entry_validation.py, every call is rejected by the host-side checks before any device access (the
buffers are host memory).  Status 2 is RNNT_STATUS_INVALID_VALUE; 3 is what the CPU location returns, so a call
that returns 3 passed every argument check."""
import ctypes as C
import math

import pytest
import torch

FULL = "acts grads labels ylen xlen V N costs scale gopt"
BWD = "acts grads labels ylen xlen V N svec scale gopt"
# name -> (parameters, the entry without lattice options and its parameters, pointers that may be NULL)
ENTRIES = {
    "rnnt_b200_loss_async_lat": ("dtype layout " + FULL + " lopt ws opt",
                                 ("rnnt_b200_loss_async_ex", "dtype layout " + FULL + " ws opt"), {"grads"}),
    "rnnt_b200_forward_lat": ("dtype acts labels ylen xlen V N costs prep lopt ws opt",
                              ("rnnt_b200_forward_16", "dtype acts labels ylen xlen V N costs prep ws opt"), set()),
    "rnnt_b200_backward_lat": ("dtype " + BWD + " lopt ws opt",
                               ("rnnt_b200_backward_ex", "dtype " + BWD + " ws opt"), {"svec"}),
    "rnnt_b200_pruned_loss_async_lat": (
        "dtype layout acts grads ranges R labels ylen xlen V N costs scale gopt lopt ws opt",
        ("rnnt_b200_pruned_loss_async_ex", "dtype layout acts grads ranges R labels ylen xlen V N costs scale gopt ws opt"),
        {"grads"}),
    "rnnt_b200_pruned_forward_lat": (
        "dtype acts ranges R labels ylen xlen V N costs prep lopt ws opt",
        ("rnnt_b200_pruned_forward", "dtype acts ranges R labels ylen xlen V N costs prep ws opt"), set()),
    "rnnt_b200_pruned_backward_lat": (
        "dtype acts grads ranges R labels ylen xlen V N svec scale gopt lopt ws opt",
        ("rnnt_b200_pruned_backward_ex", "dtype acts grads ranges R labels ylen xlen V N svec scale gopt ws opt"),
        {"svec"}),
    "rnnt_b200_add_joint_forward_lat": (
        "f g labels ylen xlen V N costs prep smooth lopt ws opt",
        ("rnnt_b200_add_joint_smoothed_forward", "f g labels ylen xlen V N costs prep smooth ws opt"), set()),
}
ACCEPTED = {
    "rnnt_b200_loss_async_lat": {(0, 0), (0, 1), (3, 0), (3, 1), (1, 0), (2, 0)},
    "rnnt_b200_forward_lat": {(0, None), (1, None), (2, None), (3, None)},
    "rnnt_b200_backward_lat": {(0, None), (1, None), (2, None), (3, None)},
    "rnnt_b200_pruned_loss_async_lat": {(0, 0), (1, 0), (2, 0), (3, 0)},
    "rnnt_b200_pruned_forward_lat": {(0, None), (1, None), (2, None), (3, None)},
    "rnnt_b200_pruned_backward_lat": {(0, None), (1, None), (2, None), (3, None)},
}
BAD = [float("nan"), float("inf"), -float("inf"), -1.0, -1e-30, -0.5]


@pytest.fixture(scope="module")
def wr():
    import warprnnt_pytorch.warp_rnnt as wr
    return wr


@pytest.fixture(scope="module")
def lib(wr):
    return C.CDLL(wr.lib_path())


class Caller:
    """Calls one entry with host buffers and otherwise valid arguments, overridden by keyword."""

    def __init__(self, wr, lib, name, params):
        from warprnnt_pytorch.joint import rnntSmoothOptions
        self.wr, self.name = wr, name
        self.params = params.split()
        types = {"dtype": C.c_int, "layout": C.c_int, "V": C.c_int, "N": C.c_int, "prep": C.c_int, "R": C.c_int,
                 "scale": C.c_float if "joint" in name else C.c_double, "gopt": wr.rnntGradOptions,
                 "lopt": wr.rnntLatticeOptions, "smooth": rnntSmoothOptions, "opt": wr.rnntOptions}
        self.pointers = [q for q in self.params if q not in types]
        self.fn = getattr(lib, name)
        self.fn.restype = C.c_int
        self.fn.argtypes = [types.get(q, C.c_void_p) for q in self.params]
        self.smooth = rnntSmoothOptions
        self.buf = (C.c_double * 64)()
        self.ibuf = (C.c_int * 8)(1, 1, 1, 1, 1, 1, 1, 1)

    def __call__(self, loc=1, maxT=2, maxU=2, blank=0, lam=0.0, **kw):
        opt = self.wr.rnntOptions(loc=loc, num_threads=0, stream=None, blank_label=blank, maxT=maxT, maxU=maxU,
                                  batch_first=True)
        args = dict(dtype=1 if self.name == "rnnt_b200_forward_16" else 0, layout=0, V=4, N=1, prep=1, R=2,
                    scale=1.0, gopt=self.wr.rnntGradOptions(0.0, 0.0), lopt=self.wr.rnntLatticeOptions(lam),
                    smooth=self.smooth(0.0, 0.0), opt=opt)
        for q in self.pointers:
            args[q] = C.addressof(self.ibuf if q in ("labels", "ylen", "xlen", "ranges") else self.buf)
        kw = {k: v for k, v in kw.items() if k in self.params}   # the old entries lack `lopt`
        args.update(kw)
        return self.fn(*[args[q] for q in self.params])


@pytest.fixture(params=sorted(ENTRIES), scope="module")
def pair(request, wr, lib):
    params, (old, old_params), _ = ENTRIES[request.param]
    return Caller(wr, lib, request.param, params), Caller(wr, lib, old, old_params)


def test_entries_exist(wr):
    for name in ENTRIES:
        getattr(wr.lib(), name)


def test_rejects_bad_penalty_before_device_access(pair):
    new, _ = pair
    for lam in BAD:
        assert new(lam=lam) == 2, lam
        assert new(loc=0, lam=lam) == 2, lam          # checked before the location
        assert new(loc=0, lam=lam, N=0) == 2, lam
    for lam in (0.0, 1e-30, 0.5, 3.0e38):
        assert new(loc=0, lam=lam) == 3, lam          # valid values reach the location check


CASES = [{}, {"V": 0}, {"V": -1}, {"N": 0}, {"N": -2}, {"maxT": 0}, {"maxU": -1}, {"blank": -1}, {"blank": 4},
         {"maxU": 1025}, {"N": 2, "maxT": 1 << 20, "maxU": 1024}, {"R": 0}, {"R": -1},
         {"N": 2, "maxT": 1 << 20, "R": 1 << 10}, {"layout": 1}, {"layout": 2}, {"dtype": 4}, {"dtype": -1},
         {"gopt": "nan"}, {"gopt": "neg"}]


@pytest.mark.parametrize("loc", [0, 1, 2])
def test_zero_penalty_takes_the_old_entry_checks(pair, loc):
    """lambda = 0 through a new entry gets exactly the status of the entry without lattice options; a valid
    lambda > 0 too."""
    new, old = pair
    for lam in (0.0, 0.25):
        for kw in CASES:
            kw = dict(kw)
            if kw.get("gopt") == "nan":
                kw["gopt"] = new.wr.rnntGradOptions(float("nan"), 0.0)
            elif kw.get("gopt") == "neg":
                kw["gopt"] = new.wr.rnntGradOptions(-1.0, 0.0)
            if "dtype" in kw and "dtype" not in new.params:
                continue
            if old.name == "rnnt_b200_forward_16" and "dtype" not in kw:
                kw["dtype"] = 1       # the old forward entry with a dtype takes 16-bit codes only
            assert new(loc=loc, lam=lam, **kw) == old(loc=loc, **kw), (lam, kw)


def test_null_pointers(pair):
    new, _ = pair
    optional = ENTRIES[new.name][2]
    for q in new.pointers:
        if q not in optional:
            assert new(**{q: None}) == 2, q
            assert new(loc=0, lam=0.5, **{q: None}) == 2, q


@pytest.mark.parametrize("name", sorted(ACCEPTED))
def test_dtype_and_layout_codes(wr, lib, name):
    call = Caller(wr, lib, name, ENTRIES[name][0])
    for dtype in range(-1, 6):
        for layout in (range(-1, 4) if "layout" in call.params else [None]):
            kw = {"dtype": dtype}
            if layout is not None:
                kw["layout"] = layout
            want = 3 if (dtype, layout) in ACCEPTED[name] else 2
            assert call(loc=0, lam=0.5, **kw) == want, kw


def test_joint_forward_smoothing_rules(wr, lib):
    call = Caller(wr, lib, "rnnt_b200_add_joint_forward_lat", ENTRIES["rnnt_b200_add_joint_forward_lat"][0])
    for lm, am in ((-0.1, 0.0), (0.0, float("nan")), (0.7, 0.7)):
        assert call(loc=0, lam=0.5, smooth=call.smooth(lm, am)) == 2
    for lm, am in ((0.0, 0.0), (0.25, 0.0), (0.25, 0.1)):
        assert call(loc=0, lam=0.5, smooth=call.smooth(lm, am)) == 3
    assert call(maxT=1 << 16, maxU=2, V=1 << 15, lam=0.5) == 2     # the joint's 32-bit factor offsets


# ---- Python keyword ----------------------------------------------------------------------------------------------
def _cpu_inputs():
    acts = torch.zeros(2, 3, 2, 5)
    labels = torch.ones(2, 1, dtype=torch.int32)
    lens = torch.full((2,), 3, dtype=torch.int32)
    ylens = torch.ones(2, dtype=torch.int32)
    return acts, labels, lens, ylens


def _callers():
    import warprnnt_pytorch as wp
    from warprnnt_pytorch import joint, pruned, warp_rnnt
    from warprnnt_pytorch.distributed import ShardedRNNTLoss
    acts, labels, lens, ylens = _cpu_inputs()
    trans, pred = torch.zeros(2, 3, 5), torch.zeros(2, 2, 5)
    ranges = torch.zeros(2, 3, dtype=torch.int32)
    costs = torch.zeros(2)
    return {
        "rnnt_loss": lambda lam: wp.rnnt_loss(acts, labels, lens, ylens, delay_penalty=lam),
        "RNNTLoss": lambda lam: wp.RNNTLoss(delay_penalty=lam),
        "ShardedRNNTLoss": lambda lam: ShardedRNNTLoss(delay_penalty=lam),
        "gpu_rnnt_async": lambda lam: warp_rnnt.gpu_rnnt_async(acts, labels, lens, ylens, costs, None, 0,
                                                               delay_penalty=lam),
        "gpu_rnnt_async_tunv": lambda lam: warp_rnnt.gpu_rnnt_async_tunv(acts, labels, lens, ylens, costs, None, 0,
                                                                         delay_penalty=lam),
        "gpu_rnnt_forward": lambda lam: warp_rnnt.gpu_rnnt_forward(acts, labels, lens, ylens, costs, 0,
                                                                   delay_penalty=lam),
        "gpu_rnnt_backward": lambda lam: warp_rnnt.gpu_rnnt_backward(acts, labels, lens, ylens, acts, None, 0, 1.0,
                                                                     None, delay_penalty=lam),
        "pruned_rnnt_loss": lambda lam: pruned.pruned_rnnt_loss(acts, labels, lens, ylens, ranges, delay_penalty=lam),
        "PrunedRNNTLoss": lambda lam: pruned.PrunedRNNTLoss(delay_penalty=lam),
        "add_joint_rnnt_loss": lambda lam: joint.add_joint_rnnt_loss(trans, pred, labels, lens, ylens,
                                                                     delay_penalty=lam),
        "AddJointRNNTLoss": lambda lam: joint.AddJointRNNTLoss(delay_penalty=lam),
        "add_joint_rnnt_loss_with_ranges": lambda lam: pruned.add_joint_rnnt_loss_with_ranges(
            trans, pred, labels, lens, ylens, 2, delay_penalty=lam),
    }


@pytest.mark.parametrize("name", sorted(_callers()))
@pytest.mark.parametrize("lam", BAD + [3.5e38])
def test_python_rejects_bad_penalty(name, lam):
    """ValueError before any other check (the tensors here are on the CPU, which would be the next error)."""
    with pytest.raises(ValueError, match="delay_penalty"):
        _callers()[name](lam)


def test_python_keyword_only():
    import warprnnt_pytorch as wp
    from warprnnt_pytorch import joint, pruned
    acts, labels, lens, ylens = _cpu_inputs()
    with pytest.raises(TypeError):
        wp.rnnt_loss(acts, labels, lens, ylens, 0, 'mean', 0.0, -1.0, 0.5)
    with pytest.raises(TypeError):
        wp.RNNTLoss(0, 'mean', 0.0, -1.0, 0.5)
    with pytest.raises(TypeError):
        pruned.PrunedRNNTLoss(0, 'mean', 0.0, -1.0, 0.5)
    with pytest.raises(TypeError):
        joint.AddJointRNNTLoss(0, 'mean', 0.0, None, 0.0, 0.0, 0.5)
    assert wp.RNNTLoss(delay_penalty=0.5).delay_penalty == 0.5
    assert pruned.PrunedRNNTLoss(delay_penalty=0.5).delay_penalty == 0.5
    assert joint.AddJointRNNTLoss(delay_penalty=0.5).delay_penalty == 0.5


def test_lattice_options_helper(wr):
    assert wr.lattice_options(0.0) is None and wr.lattice_options(0) is None
    o = wr.lattice_options(0.25)
    assert isinstance(o, wr.rnntLatticeOptions) and o.delay_penalty == 0.25
    assert C.sizeof(wr.rnntLatticeOptions) == 4
    assert math.isclose(wr.lattice_options(1e-3).delay_penalty, 1e-3, rel_tol=1e-7)
