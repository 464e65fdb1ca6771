"""Argument rules of the factor-level entries of the C-ABI (rnnt_b200_lattice_forward / _backward / _align and
rnnt_b200_lattice_workspace_size) and of the Python functions, without a GPU.

As in test_align_entries.py, every call is rejected by the host-side checks before any device access (the buffers
are host memory).  Status 2 is RNNT_STATUS_INVALID_VALUE; 3 is what the CPU location returns, so a call that
returns 3 passed every argument check."""
import ctypes as C

import pytest
import torch

import test_modified_entries as me

ENTRIES = {
    "rnnt_b200_lattice_forward": "dtype px py ylen xlen N topo costs prep ws opt",
    "rnnt_b200_lattice_backward": "dtype pxg pyg ylen xlen N topo gcosts scale ws opt",
    "rnnt_b200_lattice_align": "dtype px py ylen xlen N topo frames scores ws opt",
}
OPTIONAL = {"gcosts"}                        # NULL: all ones
NO_LABELS = {"px", "pxg", "frames"}          # no element when maxU == 1


@pytest.fixture(scope="module")
def wr():
    import warprnnt_pytorch.warp_rnnt as wr
    return wr


@pytest.fixture(scope="module")
def lib(wr):
    return C.CDLL(wr.lib_path())


@pytest.fixture(params=sorted(ENTRIES), scope="module")
def entry(request, wr, lib):
    return me.Caller(wr, lib, request.param, ENTRIES[request.param])


def test_entries_exist(wr):
    for name in list(ENTRIES) + ["rnnt_b200_lattice_workspace_size"]:
        getattr(wr.lib(), name)


def test_valid_arguments_reach_the_location_check(entry):
    for dtype in (0, 1, 2, 3):
        for topo in (0, 1):
            assert entry(loc=0, dtype=dtype, topo=topo) == 3, (dtype, topo)
    assert entry(loc=0, maxT=1, maxU=1) == 3
    assert entry(loc=0, maxU=1024) == 3
    assert entry(loc=0, blank=-1) == 3        # the blank index is not read
    assert entry(loc=0, blank=1 << 20) == 3
    if "prep" in entry.params:
        assert entry(loc=0, prep=0) == 3
    if "gcosts" in entry.params:
        assert entry(loc=0, gcosts=None) == 3


def test_dtype_and_topology(entry):
    for dtype in (-1, 4, 100):
        assert entry(loc=0, dtype=dtype) == 2, dtype
        assert entry(dtype=dtype) == 2, dtype
    for topo in me.BAD:
        assert entry(loc=0, topo=topo) == 2, topo
        assert entry(topo=topo) == 2, topo


def test_null_pointers(entry):
    for q in entry.pointers:
        if q in OPTIONAL:
            continue
        assert entry(loc=0, **{q: None}) == 2, q
        assert entry(loc=1, **{q: None}) == 2, q
        expect = 3 if q in NO_LABELS else 2
        assert entry(loc=0, maxU=1, **{q: None}) == expect, q


def test_extents(entry):
    """Rejected at the GPU location too, so before any device access (the buffers are host memory)."""
    for kw in (dict(N=0), dict(N=-1), dict(maxT=0), dict(maxT=-3), dict(maxU=0), dict(maxU=1025), dict(loc=7),
               dict(N=1 << 10, maxT=1 << 11, maxU=1 << 10)):   # N maxT maxU >= 2^31
        assert entry(loc=kw.pop("loc", 1), **kw) == 2, kw


def test_workspace_size(wr, lib):
    fn = lib.rnnt_b200_lattice_workspace_size
    fn.restype = C.c_int
    fn.argtypes = [C.c_int, C.c_int, C.c_int, C.c_size_t, C.POINTER(C.c_size_t)]
    n = C.c_size_t(0)
    for bad in ((0, 2, 1), (2, 0, 1), (2, 2, 0), (-1, 2, 1)):
        assert fn(*bad, 4, C.byref(n)) == 2, bad
    assert fn(2, 2, 1, 4, None) == 2
    sizes = {}
    for T, U, N, esz in ((1, 1, 1, 4), (150, 21, 8, 4), (150, 21, 8, 8), (150, 21, 8, 2), (1500, 301, 4, 4)):
        assert fn(T, U, N, esz, C.byref(n)) == 0
        sizes[(T, U, N, esz)] = n.value
        # factors 16 B, two lattices 8 B each per cell of the diagonal-major block
        assert n.value >= N * (T + U - 1) * U * 32
    assert sizes[(150, 21, 8, 2)] == sizes[(150, 21, 8, 4)]   # any size but 8 is the fp32 arithmetic
    assert wr.lattice_workspace_size(150, 21, 8) == sizes[(150, 21, 8, 4)]
    # no per-row statistics: smaller than the logits workspace of the same lattice
    assert sizes[(150, 21, 8, 4)] < wr.workspace_size(150, 21, 8, 4)


def _inputs(N=2, S=2, T=4, dtype=torch.float32):
    px = torch.zeros(N, S, T, dtype=dtype)
    py = torch.zeros(N, S + 1, T, dtype=dtype)
    tl = torch.full((N,), T, dtype=torch.int32)
    ul = torch.full((N,), S, dtype=torch.int32)
    return px, py, tl, ul


def test_python_surface():
    import inspect

    import warprnnt_pytorch as wp
    assert {"rnnt_lattice_loss", "RNNTLatticeLoss", "rnnt_lattice_forced_align"} <= set(wp.__all__)
    for fn in (wp.rnnt_lattice_loss, wp.rnnt_lattice_forced_align, wp.RNNTLatticeLoss):
        p = inspect.signature(fn).parameters
        assert p["rnnt_type"].kind is inspect.Parameter.KEYWORD_ONLY and p["rnnt_type"].default == "regular"
    assert inspect.signature(wp.rnnt_lattice_loss).parameters["reduction"].default == "mean"
    for name in ("gpu_lattice_forward", "gpu_lattice_backward", "gpu_lattice_align"):
        assert callable(getattr(wp.warp_rnnt, name))


@pytest.mark.parametrize("kind", ["loss", "align"])
def test_python_argument_checks(kind):
    import warprnnt_pytorch as wp
    px, py, tl, ul = _inputs()

    def call(x=px, y=py, t=tl, u=ul, **kw):
        if kind == "loss":
            return wp.rnnt_lattice_loss(x, y, t, u, **kw)
        kw.pop("reduction", None)
        return wp.rnnt_lattice_forced_align(x, y, t, u, **kw)
    for bad in ("constrained", "Regular", 1, None):
        with pytest.raises(ValueError):
            call(rnnt_type=bad)
    if kind == "loss":
        with pytest.raises(ValueError):
            call(reduction="avg")
        with pytest.raises(ValueError):
            wp.RNNTLatticeLoss(reduction="avg")
        with pytest.raises(ValueError):
            wp.RNNTLatticeLoss(rnnt_type="constrained")
    with pytest.raises(TypeError):
        call(x=px.double())                        # px and py of different dtypes
    with pytest.raises(TypeError):
        call(x=px.long(), y=py.long())             # not floating
    with pytest.raises(TypeError):
        call(t=tl.long())
    with pytest.raises(TypeError):
        call(u=ul.float())
    with pytest.raises(ValueError):
        call(x=px[0])                              # not 3-D
    with pytest.raises(ValueError):
        call(y=py[:, :2])                          # py must be [N, S+1, T]
    with pytest.raises(ValueError):
        call(y=py[..., :3])
    with pytest.raises(ValueError):
        call(x=px[..., :0], y=py[..., :0])         # no frame
    with pytest.raises(ValueError):
        call(t=tl[:1])                             # one length per utterance
    with pytest.raises(ValueError):
        call(u=ul[:1])
    with pytest.raises(ValueError):
        call(t=torch.full((2, 2), 4, dtype=torch.int32)[:, 0])   # not contiguous
    with pytest.raises(RuntimeError):              # CPU tensors: no host path
        call()
    with pytest.raises(RuntimeError):              # non-contiguous factors are copied, not refused
        call(x=px.transpose(1, 2).contiguous().transpose(1, 2))
