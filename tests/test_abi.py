"""CPU-side checks of the drop-in boundary: libwarprnnt.so loads, exports every symbol that
include/rnnt.h declares, keeps the reference's struct layout / status strings / argument
validation (src/rnnt_entrypoint.cpp:18-35,49-59,96-105).  No kernel is launched here."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rnnt.h")


@pytest.fixture(scope="module")
def wr():
    import warprnnt_pytorch.warp_rnnt as wr
    return wr


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = re.findall(r"^\s*(?:rnntStatus_t|int|void|const char\*)\s+(\w+)\s*\(", src, flags=re.M)
    return sorted(set(names))


def test_header_declares_reference_entry_points():
    syms = declared_symbols()
    for s in ("compute_rnnt_loss", "compute_rnnt_loss_fp64", "get_workspace_size",
              "get_warprnnt_version", "rnntGetStatusString", "get_rnnt_workspace_size"):
        assert s in syms


def test_library_exports_every_declared_symbol(wr):
    out = subprocess.run(["nm", "-D", "--defined-only", wr.lib_path()], capture_output=True, text=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    for s in declared_symbols():
        assert s in exported, s
        getattr(wr.lib(), s)


def test_header_compiles_as_c_and_cxx(tmp_path):
    for comp, ext, std in (("/usr/bin/gcc", "c", "-std=c11"), ("/usr/bin/g++", "cpp", "-std=c++11")):
        src = tmp_path / ("t." + ext)
        src.write_text('#include "rnnt.h"\nint main(void){ struct rnntOptions o; '
                       'return sizeof(o) == 32 ? 0 : 1; }\n')
        exe = tmp_path / ("t_" + ext)
        subprocess.check_call([comp, std, "-I", os.path.join(ROOT, "include"), str(src), "-c", "-o", str(exe)])


def test_options_struct_layout(wr):
    o = wr.rnntOptions
    assert C.sizeof(o) == 32
    offs = [getattr(o, f).offset for f, _ in o._fields_]
    assert offs == [0, 4, 8, 16, 20, 24, 28]     # SURVEY §8(a1)


def test_version_and_status_strings(wr):
    lib = wr.lib()
    assert lib.get_warprnnt_version() == 1        # tests/test_cpu.cpp:382-385 aborts otherwise
    want = {0: "no error", 1: "cuda memcpy or memset failed", 2: "invalid value",
            3: "execution failed", 4: "unknown error", 77: "unknown error"}
    for k, v in want.items():
        assert wr.status_string(k) == v


def test_workspace_size_rules(wr):
    lib = wr.lib()
    n = C.c_size_t(123)
    for bad in ((0, 3, 2), (4, 0, 2), (4, 3, 0), (-1, 3, 2)):
        assert lib.get_workspace_size(bad[0], bad[1], bad[2], True, C.byref(n), 4) == 2
    assert lib.get_workspace_size(4, 3, 2, True, C.byref(n), 4) == 0
    small = n.value
    assert lib.get_rnnt_workspace_size(4, 3, 2, True, C.byref(n), 4) == 0 and n.value == small
    assert lib.get_workspace_size(150, 21, 128, True, C.byref(n), 4) == 0
    rows = 150 * 21 * 128
    assert n.value >= rows * (2 * 4 + 2 * 4 + 8 + 8)      # stat + lp2 + alpha + beta
    assert lib.get_workspace_size(150, 21, 128, True, C.byref(n), 8) == 0
    assert n.value >= rows * (2 * 8 + 2 * 8 + 8 + 8)
    # CPU sizing keeps the reference formula (src/rnnt_entrypoint.cpp:110-118)
    assert lib.get_workspace_size(4, 3, 2, False, C.byref(n), 4) == 0 and n.value == 4 * 4 * 3 * 2 * 4


def test_argument_validation_without_gpu(wr):
    """Null pointers / non-positive sizes -> INVALID_VALUE before any CUDA call
    (src/rnnt_entrypoint.cpp:49-59); loc == RNNT_CPU -> EXECUTION_FAILED (no CPU path)."""
    lib = wr.lib()
    buf = (C.c_float * 64)()
    ibuf = (C.c_int * 8)(1, 1, 1, 1, 1, 1, 1, 1)
    p, ip = C.addressof(buf), C.addressof(ibuf)
    opt = wr.rnntOptions(loc=1, num_threads=0, stream=None, blank_label=0, maxT=2, maxU=2, batch_first=True)
    f = lib.compute_rnnt_loss
    assert f(None, None, ip, ip, ip, 4, 1, p, p, opt) == 2
    assert f(p, None, None, ip, ip, 4, 1, p, p, opt) == 2
    assert f(p, None, ip, None, ip, 4, 1, p, p, opt) == 2
    assert f(p, None, ip, ip, None, 4, 1, p, p, opt) == 2
    assert f(p, None, ip, ip, ip, 4, 1, None, p, opt) == 2
    assert f(p, None, ip, ip, ip, 4, 1, p, None, opt) == 2
    assert f(p, None, ip, ip, ip, 0, 1, p, p, opt) == 2
    assert f(p, None, ip, ip, ip, 4, 0, p, p, opt) == 2
    bad = wr.rnntOptions(loc=1, maxT=0, maxU=2)
    assert f(p, None, ip, ip, ip, 4, 1, p, p, bad) == 2
    bad = wr.rnntOptions(loc=7, maxT=2, maxU=2)
    assert f(p, None, ip, ip, ip, 4, 1, p, p, bad) == 2       # unknown location (:90-92)
    cpu = wr.rnntOptions(loc=0, maxT=2, maxU=2, batch_first=True)
    assert f(p, None, ip, ip, ip, 4, 1, p, p, cpu) == 3       # no CPU fallback
    assert lib.compute_rnnt_loss_fp64(None, None, ip, ip, ip, 4, 1, p, p, opt) == 2


def test_operator_rejects_cpu_tensors_and_bad_inputs():
    import torch
    from warprnnt_pytorch import RNNTLoss, rnnt_loss, certify_inputs
    acts = torch.zeros(1, 2, 3, 5)
    labels = torch.tensor([[1, 2]], dtype=torch.int32)
    tl = torch.tensor([2], dtype=torch.int32)
    ul = torch.tensor([2], dtype=torch.int32)
    with pytest.raises(RuntimeError):
        RNNTLoss()(acts, labels, tl, ul)          # no CPU fallback
    with pytest.raises(TypeError):
        rnnt_loss(acts, labels.long(), tl, ul)
    with pytest.raises(ValueError):
        rnnt_loss(acts, labels, torch.tensor([3], dtype=torch.int32), ul)     # T mismatch
    with pytest.raises(ValueError):
        rnnt_loss(acts, labels, tl, torch.tensor([1], dtype=torch.int32))     # U mismatch
    with pytest.raises(ValueError):
        rnnt_loss(acts[0], labels, tl, ul)        # not 4-D / batch mismatch
    with pytest.raises(ValueError):
        rnnt_loss(acts.transpose(1, 2), labels, tl, ul)   # not contiguous
    certify_inputs(acts, labels, tl, ul)


def test_dispatch_policy_matches_the_design_notes(wr):
    """Host-side shape policy (DESIGN.md 2-4): the values the H100 measurements in DESIGN.md were taken with."""
    lib = wr.lib()
    lib.rnnt_b200_debug_policy.restype = C.c_int
    lib.rnnt_b200_debug_policy.argtypes = [C.c_int, C.c_int, C.c_int]
    f = lib.rnnt_b200_debug_policy
    # chunk kernels: two lanes per row for the README short-vocabulary shapes, bank-aware (slice-major) mapping
    assert f(0, 28, 4) == 2 and f(0, 50, 4) == 2 and f(0, 100, 4) == 4 and f(0, 29, 4) == 1
    assert f(0, 129, 4) == 0 and f(0, 5000, 4) == 0 and f(0, 64, 8) == 2 and f(0, 65, 8) == 0
    assert f(1, 50, 4) == 1 and f(1, 28, 4) == 0     # V=28 with two lanes per row is conflict-free either way
    # wavefront: one warp up to 64 labels (two columns per lane from 33), one column per lane beyond
    assert [f(2, u, 0) for u in (1, 21, 32, 33, 41, 64, 65, 301, 1024)] == [1, 1, 1, 2, 2, 2, 1, 1, 1]
    assert [f(3, u, 0) for u in (21, 32, 33, 64, 65, 301, 1024)] == [32, 32, 32, 32, 96, 320, 1024]
    # factor ring: 8 diagonals alone, deeper next to streaming passes while ~100 KB allow
    assert f(4, 301, 0) == 8 and f(4, 301, 1) == 16 and f(4, 1024, 1) == 8 and f(4, 41, 1) == 8
    assert f(5, 5000, 0) == 15 and f(5, 28, 0) == 1
    assert f(99, 0, 0) == -1
