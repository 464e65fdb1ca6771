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
}
JOINTS = [n for n in ENTRIES if "add_joint" in n]
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
        params, scale_t, self.optional = ENTRIES[name]
        self.params = params.split()
        types = {"dtype": C.c_int, "layout": C.c_int, "V": C.c_int, "N": C.c_int, "prep": C.c_int,
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
        args = dict(dtype=1 if self.name.endswith("_16") else 0, layout=0, V=4, N=1, prep=1, scale=1.0,
                    gopt=self.wr.rnntGradOptions(0.0, 0.0), opt=opt)
        for q in self.pointers:
            args[q] = C.addressof(self.ibuf if q in ("labels", "ylen", "xlen") else self.buf)
        assert set(kw) <= set(self.params), kw       # an ignored override would make a valid call
        args.update(kw)
        return self.fn(*[args[q] for q in self.params])


@pytest.fixture(params=sorted(ENTRIES), scope="module")
def call(request, wr, lib):
    return Caller(wr, lib, request.param)


def test_every_compute_entry_is_listed(wr):
    assert len(ENTRIES) == 19
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
