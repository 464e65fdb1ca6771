"""Argument rules of every compute entry of the C-ABI, without a GPU.

Each call here is rejected by the host-side checks before any device access: the buffers are host
memory and must never be dereferenced.  Status 2 is RNNT_STATUS_INVALID_VALUE, 3 is
RNNT_STATUS_EXECUTION_FAILED (what a CPU location returns: there is no CPU path).  Accepted dtype and
layout codes are told apart from rejected ones by pairing them with the CPU location: an accepted code
reaches the location check (3), a rejected one stops before it (2)."""
import ctypes as C

import pytest

FULL = "acts grads labels ylen xlen V N costs scale ws opt"
FWD = "acts labels ylen xlen V N costs prep ws opt"
BWD = "acts grads labels ylen xlen V N svec scale ws opt"
JOINT = "f g dF dG labels ylen xlen V N"
PRUNED_FULL = "acts grads ranges R labels ylen xlen V N costs scale gopt ws opt"

# name -> (parameters, type of `scale`, pointers that may be NULL)
ENTRIES = {
    "compute_rnnt_loss": ("acts grads labels ylen xlen V N costs ws opt", None, {"grads"}),
    "compute_rnnt_loss_fp64": ("acts grads labels ylen xlen V N costs ws opt", None, {"grads"}),
    "compute_rnnt_loss_async": (FULL, C.c_float, {"grads"}),
    "compute_rnnt_loss_async_fp64": (FULL, C.c_double, {"grads"}),
    "rnnt_b200_forward": (FWD, None, set()),
    "rnnt_b200_forward_fp64": (FWD, None, set()),
    "rnnt_b200_backward": (BWD, C.c_float, {"svec"}),
    "rnnt_b200_backward_fp64": (BWD, C.c_double, {"svec"}),
    "rnnt_b200_loss_async_layout": ("layout " + FULL, C.c_float, {"grads"}),
    "rnnt_b200_loss_async_layout_fp64": ("layout " + FULL, C.c_double, {"grads"}),
    "rnnt_b200_loss_async_16": ("dtype " + FULL, C.c_float, {"grads"}),
    "rnnt_b200_forward_16": ("dtype " + FWD, None, set()),
    "rnnt_b200_backward_16": ("dtype " + BWD, C.c_float, {"svec"}),
    "rnnt_b200_loss_async_ex": ("dtype layout " + FULL.replace("scale", "scale gopt"), C.c_double, {"grads"}),
    "rnnt_b200_backward_ex": ("dtype " + BWD.replace("scale", "scale gopt"), C.c_double, {"svec"}),
    "rnnt_b200_add_joint_loss": (JOINT + " costs scale ws opt", C.c_float, {"dF", "dG"}),
    "rnnt_b200_add_joint_forward": ("f g labels ylen xlen V N costs prep ws opt", None, set()),
    "rnnt_b200_add_joint_backward": (JOINT + " svec scale ws opt", C.c_float, {"svec"}),
    "rnnt_b200_add_joint_backward_ex": (JOINT + " svec scale gopt ws opt", C.c_float, {"svec"}),
    "rnnt_b200_pruned_loss_async_ex": ("dtype layout " + PRUNED_FULL, C.c_double, {"grads"}),
    "rnnt_b200_pruned_forward": ("dtype acts ranges R labels ylen xlen V N costs prep ws opt", None, set()),
    "rnnt_b200_pruned_backward_ex": ("dtype acts grads ranges R labels ylen xlen V N svec scale gopt ws opt",
                                     C.c_double, {"svec"}),
}
# the (dtype, layout) codes each coded entry accepts (None: the entry has no such parameter)
ACCEPTED = {
    "rnnt_b200_loss_async_layout": {(None, 0), (None, 1)},
    "rnnt_b200_loss_async_layout_fp64": {(None, 0), (None, 1)},
    "rnnt_b200_loss_async_16": {(1, None), (2, None)},
    "rnnt_b200_forward_16": {(1, None), (2, None)},
    "rnnt_b200_backward_16": {(1, None), (2, None)},
    "rnnt_b200_loss_async_ex": {(0, 0), (0, 1), (3, 0), (3, 1), (1, 0), (2, 0)},   # TUNV only for fp32 / fp64
    "rnnt_b200_backward_ex": {(0, None), (1, None), (2, None), (3, None)},
    "rnnt_b200_pruned_loss_async_ex": {(0, 0), (1, 0), (2, 0), (3, 0)},   # [N,T,R,V] only: no TUNV layout
    "rnnt_b200_pruned_forward": {(0, None), (1, None), (2, None), (3, None)},
    "rnnt_b200_pruned_backward_ex": {(0, None), (1, None), (2, None), (3, None)},
}
# host entries outside the compute table: the pruning ranges (a kernel on an additive-joint workspace)
RANGES = {"rnnt_b200_add_joint_prune_ranges": ("ylen xlen N R ranges ws opt", None, set())}
JOINTS = [n for n in ENTRIES if "add_joint" in n]
PRUNED = [n for n in ENTRIES if "pruned" in n]
CODES = range(-1, 6)


@pytest.fixture(scope="module")
def wr():
    import warprnnt_pytorch.warp_rnnt as wr
    return wr


@pytest.fixture(scope="module")
def lib(wr):
    # a handle of our own: the argtypes set here do not leak into other tests' handles
    return C.CDLL(wr.lib_path())


class Caller:
    """Calls one entry with host buffers and otherwise valid arguments, overridden by keyword."""

    def __init__(self, wr, lib, name):
        self.wr, self.name = wr, name
        params, scale_t, self.optional = {**ENTRIES, **RANGES}[name]
        self.params = params.split()
        types = {"dtype": C.c_int, "layout": C.c_int, "V": C.c_int, "N": C.c_int, "prep": C.c_int, "R": C.c_int,
                 "scale": scale_t, "gopt": wr.rnntGradOptions, "opt": wr.rnntOptions}
        self.pointers = [q for q in self.params if q not in types]
        self.fn = getattr(lib, name)
        self.fn.restype = C.c_int
        self.fn.argtypes = [types.get(q, C.c_void_p) for q in self.params]
        self.buf = (C.c_double * 64)()
        self.ibuf = (C.c_int * 8)(1, 1, 1, 1, 1, 1, 1, 1)

    def __call__(self, loc=1, maxT=2, maxU=2, blank=0, **kw):
        opt = self.wr.rnntOptions(loc=loc, num_threads=0, stream=None, blank_label=blank, maxT=maxT, maxU=maxU,
                                  batch_first=True)
        args = dict(dtype=1 if self.name.endswith("_16") else 0, layout=0, V=4, N=1, prep=1, R=2, scale=1.0,
                    gopt=self.wr.rnntGradOptions(0.0, 0.0), opt=opt)
        for q in self.pointers:
            args[q] = C.addressof(self.ibuf if q in ("labels", "ylen", "xlen", "ranges") else self.buf)
        assert set(kw) <= set(self.params), kw       # an ignored override would make a valid call
        args.update(kw)
        return self.fn(*[args[q] for q in self.params])


@pytest.fixture(params=sorted(ENTRIES), scope="module")
def call(request, wr, lib):
    return Caller(wr, lib, request.param)


def test_every_compute_entry_is_listed(wr):
    assert len(ENTRIES) == 22
    for name in ENTRIES:
        getattr(wr.lib(), name)


def test_null_pointers(call):
    for q in call.pointers:
        if q not in call.optional:
            assert call(**{q: None}) == 2, q
            assert call(loc=0, **{q: None}) == 2, q       # pointers are checked before the location
    if "dF" in call.params:                              # the factor gradients come in pairs
        assert call(dF=None) == 2 and call(dG=None) == 2
        if call.name != "rnnt_b200_add_joint_loss":
            assert call(dF=None, dG=None) == 2         # the backward half needs them


def test_non_positive_sizes(call):
    for kw in ({"V": 0}, {"V": -1}, {"N": 0}, {"N": -3}, {"maxT": 0}, {"maxT": -1}, {"maxU": 0}, {"maxU": -2}):
        assert call(**kw) == 2, kw
        assert call(loc=0, **kw) == 2, kw                 # sizes are checked before the location


def test_locations(call):
    for loc in (2, 7, -1):
        assert call(loc=loc) == 2, loc                    # unknown location
    assert call(loc=0) == 3                               # RNNT_CPU: no CPU fallback


def test_blank_label_range(call):
    for blank in (-1, 4, 5):                              # V = 4
        assert call(blank=blank) == 2, blank
        assert call(loc=0, blank=blank) == 3, blank       # the location comes first


def test_label_extent_limit(call):
    assert call(maxU=1025) == 2
    assert call(loc=0, maxU=1025) == 3


def test_cell_count_limit(call):
    assert call(N=2, maxT=1 << 20, maxU=1024) == 2        # N * maxT * maxU == 2^31
    assert call(N=1, maxT=(1 << 31) - 1, maxU=2) == 2
    assert call(loc=0, N=2, maxT=1 << 20, maxU=1024) == 3


@pytest.mark.parametrize("name", JOINTS)
def test_joint_factor_offset_limit(wr, lib, name):
    call = Caller(wr, lib, name)
    assert call(maxT=1 << 16, maxU=2, V=1 << 15) == 2     # maxT * V == 2^31: past 32-bit factor offsets
    assert call(maxT=2, maxU=1 << 10, V=1 << 21) == 2     # maxU * V == 2^31


def test_joint_rejects_a_clamp(wr, lib):
    call = Caller(wr, lib, "rnnt_b200_add_joint_backward_ex")
    for clamp in (1.0, -1.0, 1e-30):
        assert call(loc=0, gopt=wr.rnntGradOptions(0.0, clamp)) == 2
    assert call(loc=0, gopt=wr.rnntGradOptions(0.5, 0.0)) == 3


@pytest.mark.parametrize("name", sorted(ACCEPTED))
def test_dtype_and_layout_codes(wr, lib, name):
    call = Caller(wr, lib, name)
    for dtype in (CODES if "dtype" in call.params else [None]):
        for layout in (CODES if "layout" in call.params else [None]):
            kw = {k: v for k, v in (("dtype", dtype), ("layout", layout)) if v is not None}
            want = 3 if (dtype, layout) in ACCEPTED[name] else 2
            assert call(loc=0, **kw) == want, kw


@pytest.mark.parametrize("name", PRUNED)
def test_pruned_window_rules(wr, lib, name):
    call = Caller(wr, lib, name)
    assert call(ranges=None) == 2 and call(loc=0, ranges=None) == 2
    for r in (0, -1, -2 ** 31):                           # R = s_range, rows per frame
        assert call(R=r) == 2, r
        assert call(loc=0, R=r) == 2, r                   # checked before the location
    assert call(loc=0, R=1) == 3                          # one row per frame
    assert call(loc=0, R=1000, maxU=2) == 3               # windows wider than the lattice
    # N * maxT * R rows are counted with 32 bits
    assert call(loc=0, N=2, maxT=1 << 20, R=1 << 10) == 2          # 2^31
    assert call(loc=0, N=1 << 10, maxT=1 << 11, R=1 << 10) == 2    # 2^31, another factoring
    assert call(loc=0, N=1, maxT=(1 << 31) - 1, R=1) == 3          # 2^31 - 1 reaches the location check
    assert call(loc=0, N=3, maxT=(1 << 31) // 3 // 2, R=2) == 3    # just below 2^31 (2147483646)
    if "layout" in call.params:
        assert call(loc=0, layout=1) == 2 and call(loc=0, layout=0) == 3   # [T,U,N,V] has no pruned form


def test_pruned_workspace_size(wr, lib):
    fn = lib.rnnt_b200_pruned_workspace_size
    fn.restype = C.c_int
    fn.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_size_t, C.POINTER(C.c_size_t)]

    def size(maxT=10, maxU=5, R=2, N=3, elt=4, out=True):
        n = C.c_size_t(0)
        st = fn(maxT, maxU, R, N, elt, C.byref(n) if out else None)
        return st, n.value

    st, n = size()
    assert st == 0 and n > 0
    assert size(R=1)[0] == 0 and size(R=1)[1] < n < size(R=3)[1]   # stat rows grow with R
    assert size(elt=8)[1] > n and size(elt=2) == (0, n)             # anything but 8 bytes is fp32 arithmetic
    for kw in ({"R": 0}, {"R": -1}, {"maxT": 0}, {"maxU": -1}, {"N": 0}, {"out": False}):
        assert size(**kw)[0] == 2, kw


def test_prune_ranges_rules(wr, lib):
    """rnnt_b200_add_joint_prune_ranges: every rejection is INVALID_VALUE, the CPU location included (a window
    needs the additive joint's workspace on the GPU)."""
    call = Caller(wr, lib, "rnnt_b200_add_joint_prune_ranges")
    for q in call.pointers:
        assert call(**{q: None}) == 2, q
    for kw in ({"R": 1}, {"R": 0}, {"R": -1}, {"N": 0}, {"N": -1}, {"maxT": 0}, {"maxU": 0}, {"maxU": 1025},
               {"loc": 0}, {"loc": 2}, {"loc": -1}, {"N": 2, "maxT": 1 << 20, "maxU": 1024}):
        assert call(**kw) == 2, kw
