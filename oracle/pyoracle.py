"""ctypes front-end for the CPU checkers.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module; the product package never does.

Two checkers live behind it:
  * ``oracle/librnnt_oracle.so``         our C restatement (oracle/rnnt_oracle.c)
  * ``oracle/_ref/libwarprnnt_ref_cpu.so``  the unmodified reference CPU path, compiled
    by oracle/Makefile where the reference sources are present (optional)
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE_SO = os.path.join(_HERE, "librnnt_oracle.so")
_REF_CPU_SO = os.path.join(_HERE, "_ref", "libwarprnnt_ref_cpu.so")
_REF_GPU_SO = os.path.join(_HERE, "_ref", "libwarprnnt_ref_gpu.so")

_oracle = None
_ref_cpu = None


def build(quiet=True):
    """(Re)build the checker libraries with oracle/Makefile (gcc; reference only if present)."""
    out = subprocess.run(["make", "-C", _HERE, "all"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("oracle build failed:\n" + out.stdout + out.stderr)
    if not quiet:
        print(out.stdout)


def _fp(dt):
    return C.POINTER(C.c_float if dt == np.float32 else C.c_double)


def load_oracle():
    global _oracle
    if _oracle is None:
        if not os.path.exists(_ORACLE_SO):
            build()
        _oracle = C.CDLL(_ORACLE_SO)
    return _oracle


def _ptr(a, ty):
    return a.ctypes.data_as(C.POINTER(ty)) if a is not None else None


def _prep(acts, labels, act_lens, label_lens):
    acts = np.ascontiguousarray(acts)
    assert acts.dtype in (np.float32, np.float64) and acts.ndim == 4
    labels = np.ascontiguousarray(labels, dtype=np.int32)
    act_lens = np.ascontiguousarray(act_lens, dtype=np.int32)
    label_lens = np.ascontiguousarray(label_lens, dtype=np.int32)
    N, T, U, V = acts.shape
    if labels.size == 0:  # U == 1: keep a valid pointer
        labels = np.zeros((N, 1), dtype=np.int32)
    else:
        assert labels.shape == (N, U - 1), (labels.shape, acts.shape)
    return acts, labels, act_lens, label_lens


def rnnt_logits(acts, labels, act_lens, label_lens, blank=0, want_grad=True, threads=0,
                want_lattice=False):
    """GPU convention: logits in -> (costs[N], dense grads wrt logits | None, ll_backward[N]).

    Precision follows acts.dtype (float32 mirrors the reference arithmetic; float64 = truth).
    """
    lib = load_oracle()
    acts, labels, act_lens, label_lens = _prep(acts, labels, act_lens, label_lens)
    N, T, U, V = acts.shape
    dt = acts.dtype
    cty = C.c_float if dt == np.float32 else C.c_double
    fn = lib.oracle_rnnt_logits_f32 if dt == np.float32 else lib.oracle_rnnt_logits_f64
    fn.restype = C.c_int
    costs = np.zeros(N, dtype=dt)
    llb = np.zeros(N, dtype=dt)
    grads = np.empty_like(acts) if want_grad else None
    T0, U0 = int(act_lens[0]), int(label_lens[0]) + 1
    da = np.zeros((T0, U0), dtype=dt) if want_lattice else None
    db = np.zeros((T0, U0), dtype=dt) if want_lattice else None
    rc = fn(_ptr(acts, cty), _ptr(grads, cty), _ptr(labels, C.c_int), _ptr(label_lens, C.c_int),
            _ptr(act_lens, C.c_int), C.c_int(V), C.c_int(N), C.c_int(T), C.c_int(U),
            C.c_int(blank), _ptr(costs, cty), C.c_int(threads), _ptr(da, cty), _ptr(db, cty),
            _ptr(llb, cty))
    if rc != 0:
        raise RuntimeError("oracle_rnnt_logits rc=%d" % rc)
    if want_lattice:
        return costs, grads, llb, da, db
    return costs, grads, llb


def rnnt_logprobs(log_probs, labels, act_lens, label_lens, blank=0, want_grad=True, threads=0):
    """CPU convention: log-probs in -> (costs[N], sparse grads wrt log-probs | None)."""
    lib = load_oracle()
    lp, labels, act_lens, label_lens = _prep(log_probs, labels, act_lens, label_lens)
    N, T, U, V = lp.shape
    dt = lp.dtype
    cty = C.c_float if dt == np.float32 else C.c_double
    fn = lib.oracle_rnnt_logprobs_f32 if dt == np.float32 else lib.oracle_rnnt_logprobs_f64
    fn.restype = C.c_int
    costs = np.zeros(N, dtype=dt)
    grads = np.empty_like(lp) if want_grad else None
    rc = fn(_ptr(lp, cty), _ptr(grads, cty), _ptr(labels, C.c_int), _ptr(label_lens, C.c_int),
            _ptr(act_lens, C.c_int), C.c_int(V), C.c_int(N), C.c_int(T), C.c_int(U),
            C.c_int(blank), _ptr(costs, cty), C.c_int(threads), None, None)
    if rc != 0:
        raise RuntimeError("oracle_rnnt_logprobs rc=%d" % rc)
    return costs, grads


# --------------------------------------------------------------------------------------
# The unmodified reference, through its own C-ABI (include/rnnt.h of the reference).
# --------------------------------------------------------------------------------------
class RnntOptions(C.Structure):
    """rnntOptions, 32 bytes, passed by value (reference include/rnnt.h:43-64)."""
    _fields_ = [("loc", C.c_int), ("num_threads", C.c_uint), ("stream", C.c_void_p),
                ("blank_label", C.c_int), ("maxT", C.c_int), ("maxU", C.c_int),
                ("batch_first", C.c_bool)]


def have_ref_cpu():
    return os.path.exists(_REF_CPU_SO)


def have_ref_gpu():
    return os.path.exists(_REF_GPU_SO)


def ref_gpu_path():
    return _REF_GPU_SO


def load_ref_cpu():
    global _ref_cpu
    if _ref_cpu is None:
        if not have_ref_cpu():
            return None
        _ref_cpu = C.CDLL(_REF_CPU_SO)
        assert _ref_cpu.get_warprnnt_version() == 1
    return _ref_cpu


def ref_cpu_logprobs(log_probs, labels, act_lens, label_lens, blank=0, want_grad=True, threads=0):
    """Reference compute_rnnt_loss(loc=RNNT_CPU, batch_first=true): log-probs in, sparse grads out."""
    lib = load_ref_cpu()
    if lib is None:
        raise RuntimeError("oracle/_ref/libwarprnnt_ref_cpu.so is not built")
    lp, labels, act_lens, label_lens = _prep(log_probs, labels, act_lens, label_lens)
    N, T, U, V = lp.shape
    dt = lp.dtype
    cty = C.c_float if dt == np.float32 else C.c_double
    fn = lib.compute_rnnt_loss if dt == np.float32 else lib.compute_rnnt_loss_fp64
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                   C.c_void_p, C.c_void_p, RnntOptions]
    nbytes = C.c_size_t(0)
    lib.get_workspace_size.argtypes = [C.c_int, C.c_int, C.c_int, C.c_bool,
                                       C.POINTER(C.c_size_t), C.c_size_t]
    rc = lib.get_workspace_size(T, U, N, False, C.byref(nbytes), lp.itemsize)
    assert rc == 0
    ws = np.zeros(nbytes.value, dtype=np.uint8)
    costs = np.zeros(N, dtype=dt)
    grads = np.empty_like(lp) if want_grad else None
    opt = RnntOptions(loc=0, num_threads=threads, stream=None, blank_label=blank, maxT=T, maxU=U,
                      batch_first=True)
    rc = fn(lp.ctypes.data, grads.ctypes.data if want_grad else None, labels.ctypes.data,
            label_lens.ctypes.data, act_lens.ctypes.data, V, N, costs.ctypes.data, ws.ctypes.data,
            opt)
    if rc != 0:
        raise RuntimeError("reference compute_rnnt_loss rc=%d" % rc)
    return costs, grads


# --------------------------------------------------------------------------------------
# Fixed inputs of the stored reference answers (tests/golden/make_golden.py writes them,
# the tests recompute the inputs and compare against the stored outputs).
# --------------------------------------------------------------------------------------
def det_uniform(shape, seed, device):
    """float32 values in [0, 1) from an integer hash of (flat index, seed): the same numbers on every
    device, driver and torch version, unlike a torch generator whose stream follows the launch grid."""
    import torch
    n = int(np.prod(shape))
    out = torch.empty(n, dtype=torch.float32, device=device)
    step = 1 << 26
    for s in range(0, n, step):
        x = torch.arange(s, min(n, s + step), dtype=torch.int64, device=device)
        x = (x + seed * 0x632BE5AB) & 0xFFFFFFFF
        x = (((x >> 16) ^ x) * 0x45D9F3B) & 0xFFFFFFFF
        x = (((x >> 16) ^ x) * 0x45D9F3B) & 0xFFFFFFFF
        x = (x >> 16) ^ x
        out[s:s + x.numel()] = (x >> 8).to(torch.float32) * (1.0 / (1 << 24))
    return out.view(*shape)


# name: (N, T, L, V, ragged lengths, seed) - the README shapes of the reference and the headline shape
REF_GPU_CASES = {
    "small": (8, 50, 10, 15, True, 5),
    "readme_small_vocab": (16, 150, 40, 28, True, 5),
    "readme_large_vocab_N4": (4, 150, 20, 5000, True, 5),
    "headline": (128, 150, 20, 5000, False, 9),
}
GRAD_SAMPLES = 512   # gradient elements stored per case, at seeded positions


def ref_gpu_case_inputs(name, device):
    """(acts [N,T,U,V] on `device`, labels, act_lens, label_lens, sampled flat gradient indices)."""
    N, T, L, V, ragged, seed = REF_GPU_CASES[name]
    acts = det_uniform((N, T, L + 1, V), seed, device)
    rng = np.random.default_rng(seed)
    labels = rng.integers(1, V, size=(N, L)).astype(np.int32)
    tl, ul = np.full(N, T, np.int32), np.full(N, L, np.int32)
    if ragged:
        tl[1::3] = rng.integers(T // 2, T + 1, size=len(tl[1::3]))
        ul[2::3] = rng.integers(0, L + 1, size=len(ul[2::3]))
    idx = np.sort(rng.integers(0, acts.numel(), size=GRAD_SAMPLES, dtype=np.int64))
    return acts, labels, tl, ul, idx


def gpu_loss(lib, workspace_bytes, acts, labels, act_lens, label_lens, opt_type):
    """compute_rnnt_loss(loc=GPU) of a C-ABI library `lib` (this project's or the reference's) on device
    tensors; returns (costs as numpy float32, gradient tensor pre-filled with NaN)."""
    import torch
    dev = acts.device
    N, T, U, V = acts.shape
    lab, tl, ul = (torch.as_tensor(x).to(dev) for x in (labels, act_lens, label_lens))
    opt = opt_type(loc=1, num_threads=0, stream=torch.cuda.current_stream(dev).cuda_stream,
                   blank_label=0, maxT=T, maxU=U, batch_first=True)
    ws = torch.empty(workspace_bytes, dtype=torch.uint8, device=dev)
    grads = torch.full_like(acts, float("nan"))
    costs = np.zeros(N, np.float32)
    st = lib.compute_rnnt_loss(acts.data_ptr(), grads.data_ptr(), lab.data_ptr(), ul.data_ptr(),
                               tl.data_ptr(), V, N, costs.ctypes.data, ws.data_ptr(), opt)
    if st != 0:
        raise RuntimeError("compute_rnnt_loss status %d" % st)
    torch.cuda.synchronize(dev)
    return costs, grads


def grad_summary(grads, idx):
    """(gradient values at the flat positions idx, per-utterance sum of squares in float64)."""
    import torch
    flat = grads.view(-1)
    at = flat[torch.as_tensor(idx, device=grads.device)].cpu().numpy()
    sumsq = np.array([float((grads[b].double() ** 2).sum()) for b in range(grads.shape[0])])
    return at, sumsq


def log_softmax_np(x):
    m = x.max(axis=-1, keepdims=True)
    return (x - m) - np.log(np.exp(x - m).sum(axis=-1, keepdims=True))


def ref_cpu_logits(acts, labels, act_lens, label_lens, blank=0, threads=0):
    """logits -> log_softmax -> reference CPU lib -> log_softmax backward (what warprnnt_pytorch
    composes on CPU, pytorch_binding/warprnnt_pytorch/__init__.py:95-98 + autograd)."""
    acts = np.ascontiguousarray(acts)
    lp = log_softmax_np(acts)
    costs, g = ref_cpu_logprobs(lp, labels, act_lens, label_lens, blank, True, threads)
    dx = g - np.exp(lp) * g.sum(axis=-1, keepdims=True)
    return costs, dx.astype(acts.dtype)
