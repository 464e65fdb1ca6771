"""Argument rules of the forced-alignment entries of the C-ABI (rnnt_b200_align, rnnt_b200_pruned_align) and of the
Python functions, without a GPU.

As in test_modified_entries.py, every call is rejected by the host-side checks before any device access (the buffers
are host memory).  Status 2 is RNNT_STATUS_INVALID_VALUE; 3 is what the CPU location returns, so a call that
returns 3 passed every argument check."""
import ctypes as C

import pytest
import torch

import test_modified_entries as me

ENTRIES = {
    "rnnt_b200_align": "dtype layout acts labels ylen xlen V N topo frames scores ws opt",
    "rnnt_b200_pruned_align": "dtype acts ranges R labels ylen xlen V N topo frames scores ws opt",
}


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
    for name in ENTRIES:
        getattr(wr.lib(), name)


def test_valid_arguments_reach_the_location_check(entry):
    for dtype in (0, 1, 2, 3):
        for topo in (0, 1):
            assert entry(loc=0, dtype=dtype, topo=topo) == 3, (dtype, topo)
    assert entry(loc=0, maxU=1, frames=None) == 3     # no labels: frames [N, 0] may be NULL
    assert entry(loc=0, maxT=1, maxU=1) == 3


def test_dtype_layout_and_topology(entry):
    for dtype in (-1, 4, 100):
        assert entry(loc=0, dtype=dtype) == 2, dtype
    for topo in me.BAD:
        assert entry(loc=0, topo=topo) == 2, topo
        assert entry(topo=topo) == 2, topo
    if "layout" in entry.params:
        assert entry(loc=0, layout=1, dtype=0) == 3
        assert entry(loc=0, layout=1, dtype=3) == 3
        for dtype in (1, 2):   # the 16-bit types have no time-major layout
            assert entry(loc=0, layout=1, dtype=dtype) == 2
        for layout in (-1, 2, 7):
            assert entry(loc=0, layout=layout) == 2, layout


def test_null_pointers(entry):
    for q in entry.pointers:
        assert entry(loc=0, **{q: None}) == 2, q


def test_extents(entry):
    """Rejected at the GPU location too, so before any device access (the buffers are host memory)."""
    for kw in (dict(N=0), dict(N=-1), dict(V=0), dict(maxT=0), dict(maxU=0), dict(maxU=1025), dict(blank=-1),
               dict(blank=4), dict(loc=7), dict(N=1 << 10, maxT=1 << 11, maxU=1 << 10)):   # N maxT maxU >= 2^31
        assert entry(loc=kw.pop("loc", 1), **kw) == 2, kw
    assert entry(loc=0, maxU=1024) == 3
    if "R" in entry.params:
        for R in (0, -1):
            assert entry(loc=0, R=R) == 2, R
        assert entry(loc=0, R=1) == 3
        assert entry(loc=0, N=1 << 10, maxT=1 << 11, R=1 << 10) == 2


def test_python_surface():
    import warprnnt_pytorch as wp
    assert {"rnnt_forced_align", "pruned_rnnt_forced_align"} <= set(wp.__all__)
    for fn in (wp.rnnt_forced_align, wp.pruned_rnnt_forced_align):
        import inspect
        p = inspect.signature(fn).parameters
        assert p["rnnt_type"].kind is inspect.Parameter.KEYWORD_ONLY and p["rnnt_type"].default == "regular"
        assert p["blank"].default == 0


def _inputs(N=2, T=4, U=3, V=5, dtype=torch.float32):
    acts = torch.zeros(N, T, U, V, dtype=dtype)
    labels = torch.ones(N, U - 1, dtype=torch.int32)
    tl = torch.full((N,), T, dtype=torch.int32)
    ul = torch.full((N,), U - 1, dtype=torch.int32)
    return acts, labels, tl, ul


@pytest.mark.parametrize("kind", ["dense", "pruned"])
def test_python_argument_checks(kind):
    import warprnnt_pytorch as wp
    acts, labels, tl, ul = _inputs()
    if kind == "dense":
        def call(a=acts, lab=labels, t=tl, u=ul, **kw):
            return wp.rnnt_forced_align(a, lab, t, u, **kw)
    else:
        ranges = torch.zeros(2, 4, dtype=torch.int32)

        def call(a=acts, lab=labels, t=tl, u=ul, **kw):
            return wp.pruned_rnnt_forced_align(a, lab, t, u, kw.pop("ranges", ranges), **kw)
    for bad in ("constrained", "Regular", 1, None):
        with pytest.raises(ValueError):
            call(rnnt_type=bad)
    with pytest.raises(TypeError):
        call(lab=labels.long())
    with pytest.raises(TypeError):
        call(t=tl.long())
    with pytest.raises(TypeError):
        call(u=ul.float())
    with pytest.raises(ValueError):
        call(a=acts[0])                            # not 4-D
    with pytest.raises(ValueError):
        call(t=tl[:1])                             # one length per utterance
    with pytest.raises(ValueError):
        call(a=acts.transpose(1, 2))               # not contiguous
    if kind == "pruned":
        with pytest.raises(ValueError):
            call(ranges=torch.zeros(2, 3, dtype=torch.int32))
        with pytest.raises(TypeError):
            call(ranges=torch.zeros(2, 4, dtype=torch.int64))
    with pytest.raises(RuntimeError):              # CPU tensors: no host path
        call()
