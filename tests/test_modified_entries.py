"""Argument rules of the topology (rnnt_type) entries of the C-ABI and of the Python keyword, without a GPU.

As in test_delay_entries.py, every call is rejected by the host-side checks before any device access (the buffers
are host memory).  Status 2 is RNNT_STATUS_INVALID_VALUE; 3 is what the CPU location returns, so a call that
returns 3 passed every argument check."""
import ctypes as C

import pytest
import torch

import test_delay_entries as de

FULL = de.FULL
BWD = de.BWD
# name -> (parameters, the entry without a topology and its parameters, pointers that may be NULL)
ENTRIES = {
    "rnnt_b200_loss_async_topo": ("dtype layout " + FULL + " lopt topo ws opt",
                                  ("rnnt_b200_loss_async_lat", "dtype layout " + FULL + " lopt ws opt"), {"grads"}),
    "rnnt_b200_forward_topo": ("dtype acts labels ylen xlen V N costs prep lopt topo ws opt",
                               ("rnnt_b200_forward_lat", "dtype acts labels ylen xlen V N costs prep lopt ws opt"),
                               set()),
    "rnnt_b200_backward_topo": ("dtype " + BWD + " lopt topo ws opt",
                                ("rnnt_b200_backward_lat", "dtype " + BWD + " lopt ws opt"), {"svec"}),
    "rnnt_b200_pruned_loss_async_topo": (
        "dtype layout acts grads ranges R labels ylen xlen V N costs scale gopt lopt topo ws opt",
        ("rnnt_b200_pruned_loss_async_lat",
         "dtype layout acts grads ranges R labels ylen xlen V N costs scale gopt lopt ws opt"), {"grads"}),
    "rnnt_b200_pruned_forward_topo": (
        "dtype acts ranges R labels ylen xlen V N costs prep lopt topo ws opt",
        ("rnnt_b200_pruned_forward_lat", "dtype acts ranges R labels ylen xlen V N costs prep lopt ws opt"), set()),
    "rnnt_b200_pruned_backward_topo": (
        "dtype acts grads ranges R labels ylen xlen V N svec scale gopt lopt topo ws opt",
        ("rnnt_b200_pruned_backward_lat",
         "dtype acts grads ranges R labels ylen xlen V N svec scale gopt lopt ws opt"), {"svec"}),
    "rnnt_b200_add_joint_forward_topo": (
        "f g labels ylen xlen V N costs prep smooth lopt topo ws opt",
        ("rnnt_b200_add_joint_forward_lat", "f g labels ylen xlen V N costs prep smooth lopt ws opt"), set()),
    "rnnt_b200_add_joint_backward_topo": (
        "f g df dg labels ylen xlen V N svec scale gopt smooth topo ws opt",
        ("rnnt_b200_add_joint_smoothed_backward", "f g df dg labels ylen xlen V N svec scale gopt smooth ws opt"),
        {"svec"}),
}
BAD = [-1, 2, 3, 100, -(1 << 31), (1 << 31) - 1]


@pytest.fixture(scope="module")
def wr():
    import warprnnt_pytorch.warp_rnnt as wr
    return wr


@pytest.fixture(scope="module")
def lib(wr):
    return C.CDLL(wr.lib_path())


class Caller(de.Caller):
    """test_delay_entries.Caller with the `topo` argument (RNNT_B200_RNNT_REGULAR unless given)."""

    def __init__(self, wr, lib, name, params):
        super().__init__(wr, lib, name, params)
        self.fn.argtypes = [C.c_int if q == "topo" else t for q, t in zip(self.params, self.fn.argtypes)]
        self.pointers = [q for q in self.pointers if q != "topo"]

    def __call__(self, topo=0, **kw):
        if "topo" in self.params:
            kw["topo"] = topo
        return super().__call__(**kw)


@pytest.fixture(params=sorted(ENTRIES), scope="module")
def pair(request, wr, lib):
    params, (old, old_params), _ = ENTRIES[request.param]
    return Caller(wr, lib, request.param, params), Caller(wr, lib, old, old_params)


def test_entries_exist(wr):
    for name in list(ENTRIES) + ["rnnt_b200_add_joint_prune_ranges_topo"]:
        getattr(wr.lib(), name)
    assert (wr.RNNT_B200_RNNT_REGULAR, wr.RNNT_B200_RNNT_MODIFIED) == (0, 1)


def test_rejects_bad_topology_before_device_access(pair):
    new, _ = pair
    for topo in BAD:
        assert new(topo=topo) == 2, topo
        assert new(loc=0, topo=topo) == 2, topo          # checked before the location
        assert new(loc=0, topo=topo, lam=0.5) == 2, topo
    for topo in (0, 1):
        assert new(loc=0, topo=topo) == 3, topo           # valid values reach the location check


@pytest.mark.parametrize("loc", [0, 1, 2])
def test_valid_topology_takes_the_old_entry_checks(pair, loc):
    """Either topology through a new entry gets exactly the status of the entry without one.  At the GPU location
    only argument sets that the old entry rejects before its location check are tried: the buffers are host memory."""
    new, old = pair
    for topo in (0, 1):
        for lam in (0.0, 0.25, -1.0):
            for kw in de.CASES:
                kw = dict(kw)
                if kw.get("gopt") == "nan":
                    kw["gopt"] = new.wr.rnntGradOptions(float("nan"), 0.0)
                elif kw.get("gopt") == "neg":
                    kw["gopt"] = new.wr.rnntGradOptions(-1.0, 0.0)
                if "dtype" in kw and "dtype" not in new.params:
                    continue
                if loc == 1 and old(loc=0, lam=lam, **kw) != 2:
                    continue
                assert new(loc=loc, lam=lam, topo=topo, **kw) == old(loc=loc, lam=lam, **kw), (topo, lam, kw)


def test_null_pointers(pair):
    new, _ = pair
    optional = ENTRIES[new.name][2]
    for q in new.pointers:
        if q not in optional:
            assert new(**{q: None}) == 2, q
            assert new(loc=0, topo=1, **{q: None}) == 2, q


def test_joint_rules(wr, lib):
    fwd = Caller(wr, lib, "rnnt_b200_add_joint_forward_topo", ENTRIES["rnnt_b200_add_joint_forward_topo"][0])
    bwd = Caller(wr, lib, "rnnt_b200_add_joint_backward_topo", ENTRIES["rnnt_b200_add_joint_backward_topo"][0])
    for call in (fwd, bwd):
        for lm, am in ((-0.1, 0.0), (0.0, float("nan")), (0.7, 0.7)):
            assert call(loc=0, topo=1, smooth=call.smooth(lm, am)) == 2
        for lm, am in ((0.0, 0.0), (0.25, 0.0), (0.25, 0.1)):
            assert call(loc=0, topo=1, smooth=call.smooth(lm, am)) == 3
    assert bwd(loc=0, topo=1, gopt=wr.rnntGradOptions(0.0, 1.0)) == 2      # no clamp on the joint
    assert bwd(loc=0, topo=1, gopt=wr.rnntGradOptions(0.5, 0.0)) == 3
    assert bwd(loc=0, topo=1, dg=None) == 2                                 # both factor gradients or neither


def test_prune_ranges_rules(wr, lib):
    fn = lib.rnnt_b200_add_joint_prune_ranges_topo
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, wr.rnntOptions]
    old = lib.rnnt_b200_add_joint_prune_ranges
    old.restype = C.c_int
    old.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, wr.rnntOptions]
    ibuf, buf = (C.c_int * 8)(1, 1, 1, 1, 1, 1, 1, 1), (C.c_double * 64)()
    p, q = C.addressof(ibuf), C.addressof(buf)

    def opt(loc=1, maxT=2, maxU=2):
        return wr.rnntOptions(loc=loc, num_threads=0, stream=None, blank_label=0, maxT=maxT, maxU=maxU,
                              batch_first=True)
    for topo in BAD:
        assert fn(p, p, 1, 2, p, q, topo, opt()) == 2, topo      # before any device query
    for topo in (0, 1):
        for args in ((p, p, 1, 2, p, q), (None, p, 1, 2, p, q), (p, p, 0, 2, p, q), (p, p, 1, 1, p, q),
                     (p, p, 1, 2, None, q), (p, p, 1, 2, p, None)):
            for o in (opt(loc=0), opt(maxU=1025), opt(maxT=0)):
                assert fn(*args, topo, o) == old(*args, o), (topo, args)


# ---- Python keyword ----------------------------------------------------------------------------------------------
def _callers():
    import warprnnt_pytorch as wp
    from warprnnt_pytorch import joint, pruned, warp_rnnt
    from warprnnt_pytorch.distributed import ShardedRNNTLoss
    acts, labels, lens, ylens = de._cpu_inputs()
    trans, pred = torch.zeros(2, 3, 5), torch.zeros(2, 2, 5)
    ranges = torch.zeros(2, 3, dtype=torch.int32)
    costs = torch.zeros(2)
    return {
        "rnnt_loss": lambda k: wp.rnnt_loss(acts, labels, lens, ylens, rnnt_type=k),
        "RNNTLoss": lambda k: wp.RNNTLoss(rnnt_type=k),
        "ShardedRNNTLoss": lambda k: ShardedRNNTLoss(rnnt_type=k),
        "gpu_rnnt_async": lambda k: warp_rnnt.gpu_rnnt_async(acts, labels, lens, ylens, costs, None, 0, rnnt_type=k),
        "gpu_rnnt_async_tunv": lambda k: warp_rnnt.gpu_rnnt_async_tunv(acts, labels, lens, ylens, costs, None, 0,
                                                                       rnnt_type=k),
        "gpu_rnnt_forward": lambda k: warp_rnnt.gpu_rnnt_forward(acts, labels, lens, ylens, costs, 0, rnnt_type=k),
        "gpu_rnnt_backward": lambda k: warp_rnnt.gpu_rnnt_backward(acts, labels, lens, ylens, acts, None, 0, 1.0,
                                                                   None, rnnt_type=k),
        "pruned_rnnt_loss": lambda k: pruned.pruned_rnnt_loss(acts, labels, lens, ylens, ranges, rnnt_type=k),
        "PrunedRNNTLoss": lambda k: pruned.PrunedRNNTLoss(rnnt_type=k),
        "add_joint_rnnt_loss": lambda k: joint.add_joint_rnnt_loss(trans, pred, labels, lens, ylens, rnnt_type=k),
        "AddJointRNNTLoss": lambda k: joint.AddJointRNNTLoss(rnnt_type=k),
        "add_joint_rnnt_loss_with_ranges": lambda k: pruned.add_joint_rnnt_loss_with_ranges(
            trans, pred, labels, lens, ylens, 2, rnnt_type=k),
    }


@pytest.mark.parametrize("name", sorted(_callers()))
@pytest.mark.parametrize("kind", ["Modified", "one_sym", "", None, 1, "regular ", "constrained"])
def test_python_rejects_bad_rnnt_type(name, kind):
    """ValueError before any other check (the tensors here are on the CPU, which would be the next error)."""
    with pytest.raises(ValueError, match="constrained' is not supported" if kind == "constrained" else "rnnt_type"):
        _callers()[name](kind)


def test_python_keyword_only():
    import warprnnt_pytorch as wp
    from warprnnt_pytorch import joint, pruned
    from warprnnt_pytorch.distributed import ShardedRNNTLoss
    acts, labels, lens, ylens = de._cpu_inputs()
    with pytest.raises(TypeError):
        wp.rnnt_loss(acts, labels, lens, ylens, 0, 'mean', 0.0, -1.0, 0.0, 'modified')
    with pytest.raises(TypeError):
        wp.RNNTLoss(0, 'mean', 0.0, -1.0, 0.0, 'modified')
    with pytest.raises(TypeError):
        pruned.PrunedRNNTLoss(0, 'mean', 0.0, -1.0, 0.0, 'modified')
    with pytest.raises(TypeError):
        joint.AddJointRNNTLoss(0, 'mean', 0.0, None, 0.0, 0.0, 0.0, 'modified')
    for cls in (wp.RNNTLoss, pruned.PrunedRNNTLoss, joint.AddJointRNNTLoss, ShardedRNNTLoss):
        assert cls().rnnt_type == 'regular'
        assert cls(rnnt_type='modified').rnnt_type == 'modified'


def test_rnnt_type_code(wr):
    assert wr.rnnt_type_code('regular') == wr.RNNT_B200_RNNT_REGULAR
    assert wr.rnnt_type_code('modified') == wr.RNNT_B200_RNNT_MODIFIED
