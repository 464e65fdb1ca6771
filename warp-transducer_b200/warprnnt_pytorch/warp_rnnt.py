"""`warprnnt_pytorch.warp_rnnt` — the extension-module surface of the reference binding
(pytorch_binding/src/binding.cpp:12-19,84-91,157-162), bound to libwarprnnt.so's C-ABI.

    gpu_rnnt(acts, labels, input_lengths, label_lengths, costs, grads, blank_label, num_threads) -> int
    cpu_rnnt(...)   raises: this build has no CPU path (and never falls back to one)

The library is loaded eagerly; a missing or unloadable libwarprnnt.so is an ImportError, not a
silent fallback.
"""
import ctypes as C
import math
import os

import torch

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB_PATH = os.environ.get("WARP_RNNT_LIB", os.path.join(_PKG, "lib", "libwarprnnt.so"))


class rnntOptions(C.Structure):
    """include/rnnt.h `struct rnntOptions` (32 bytes, by value)."""
    _fields_ = [("loc", C.c_int), ("num_threads", C.c_uint), ("stream", C.c_void_p),
                ("blank_label", C.c_int), ("maxT", C.c_int), ("maxU", C.c_int),
                ("batch_first", C.c_bool)]


class rnntGradOptions(C.Structure):
    """include/rnnt.h `struct rnntGradOptions` (8 bytes, by value; zero = both options off)."""
    _fields_ = [("fastemit_lambda", C.c_float), ("clamp", C.c_float)]


class rnntLatticeOptions(C.Structure):
    """include/rnnt.h `struct rnntLatticeOptions` (4 bytes, by value; zero = off)."""
    _fields_ = [("delay_penalty", C.c_float)]


RNNT_CPU, RNNT_GPU = 0, 1
RNNT_STATUS_SUCCESS = 0

if not os.path.exists(_LIB_PATH):
    raise ImportError(
        "libwarprnnt.so not found at %s - build it with `python warp-transducer_b200/build.py` "
        "(there is no CPU or PyTorch fallback)" % _LIB_PATH)
_lib = C.CDLL(_LIB_PATH)
assert C.sizeof(rnntOptions) == 32

_P = C.c_void_p
for _name in ("compute_rnnt_loss", "compute_rnnt_loss_fp64"):
    _f = getattr(_lib, _name)
    _f.restype = C.c_int
    _f.argtypes = [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P, rnntOptions]
_lib.compute_rnnt_loss_async.restype = C.c_int
_lib.compute_rnnt_loss_async.argtypes = [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_float, _P, rnntOptions]
_lib.compute_rnnt_loss_async_fp64.restype = C.c_int
_lib.compute_rnnt_loss_async_fp64.argtypes = [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_double, _P, rnntOptions]
for _name, _ct in (("rnnt_b200_forward", C.c_float), ("rnnt_b200_forward_fp64", C.c_double)):
    _f = getattr(_lib, _name)
    _f.restype = C.c_int
    _f.argtypes = [_P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int, _P, rnntOptions]
for _name, _ct in (("rnnt_b200_backward", C.c_float), ("rnnt_b200_backward_fp64", C.c_double)):
    _f = getattr(_lib, _name)
    _f.restype = C.c_int
    _f.argtypes = [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, _ct, _P, rnntOptions]
_lib.rnnt_b200_loss_async_16.restype = C.c_int
_lib.rnnt_b200_loss_async_16.argtypes = [C.c_int, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_float, _P, rnntOptions]
_lib.rnnt_b200_forward_16.restype = C.c_int
_lib.rnnt_b200_forward_16.argtypes = [C.c_int, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int, _P, rnntOptions]
_lib.rnnt_b200_backward_16.restype = C.c_int
_lib.rnnt_b200_backward_16.argtypes = [C.c_int, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_float, _P, rnntOptions]
RNNT_B200_BF16, RNNT_B200_FP16 = 1, 2
_lib.rnnt_b200_loss_async_layout.restype = C.c_int
_lib.rnnt_b200_loss_async_layout.argtypes = [C.c_int, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_float, _P, rnntOptions]
_lib.rnnt_b200_loss_async_layout_fp64.restype = C.c_int
_lib.rnnt_b200_loss_async_layout_fp64.argtypes = [C.c_int, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_double, _P, rnntOptions]
RNNT_B200_LAYOUT_NTUV, RNNT_B200_LAYOUT_TUNV = 0, 1
RNNT_B200_FP32, RNNT_B200_FP64 = 0, 3
_lib.rnnt_b200_loss_async_ex.restype = C.c_int
_lib.rnnt_b200_loss_async_ex.argtypes = [C.c_int, C.c_int, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_double,
                                         rnntGradOptions, _P, rnntOptions]
_lib.rnnt_b200_backward_ex.restype = C.c_int
_lib.rnnt_b200_backward_ex.argtypes = [C.c_int, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_double,
                                       rnntGradOptions, _P, rnntOptions]
_lib.rnnt_b200_loss_async_lat.restype = C.c_int
_lib.rnnt_b200_loss_async_lat.argtypes = [C.c_int, C.c_int, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_double,
                                          rnntGradOptions, rnntLatticeOptions, _P, rnntOptions]
_lib.rnnt_b200_forward_lat.restype = C.c_int
_lib.rnnt_b200_forward_lat.argtypes = [C.c_int, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int, rnntLatticeOptions,
                                       _P, rnntOptions]
_lib.rnnt_b200_backward_lat.restype = C.c_int
_lib.rnnt_b200_backward_lat.argtypes = [C.c_int, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_double,
                                        rnntGradOptions, rnntLatticeOptions, _P, rnntOptions]
RNNT_B200_RNNT_REGULAR, RNNT_B200_RNNT_MODIFIED = 0, 1
_lib.rnnt_b200_loss_async_topo.restype = C.c_int
_lib.rnnt_b200_loss_async_topo.argtypes = [C.c_int, C.c_int, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_double,
                                           rnntGradOptions, rnntLatticeOptions, C.c_int, _P, rnntOptions]
_lib.rnnt_b200_forward_topo.restype = C.c_int
_lib.rnnt_b200_forward_topo.argtypes = [C.c_int, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int, rnntLatticeOptions,
                                        C.c_int, _P, rnntOptions]
_lib.rnnt_b200_backward_topo.restype = C.c_int
_lib.rnnt_b200_backward_topo.argtypes = [C.c_int, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_double,
                                         rnntGradOptions, rnntLatticeOptions, C.c_int, _P, rnntOptions]
_lib.rnnt_b200_align.restype = C.c_int
_lib.rnnt_b200_align.argtypes = [C.c_int, C.c_int, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P, rnntOptions]
_lib.rnnt_b200_pruned_align.restype = C.c_int
_lib.rnnt_b200_pruned_align.argtypes = [C.c_int, _P, _P, C.c_int, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P,
                                        rnntOptions]
_lib.rnnt_b200_lattice_workspace_size.restype = C.c_int
_lib.rnnt_b200_lattice_workspace_size.argtypes = [C.c_int, C.c_int, C.c_int, C.c_size_t, C.POINTER(C.c_size_t)]
_lib.rnnt_b200_lattice_forward.restype = C.c_int
_lib.rnnt_b200_lattice_forward.argtypes = [C.c_int, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int, _P, rnntOptions]
_lib.rnnt_b200_lattice_backward.restype = C.c_int
_lib.rnnt_b200_lattice_backward.argtypes = [C.c_int, _P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_double, _P,
                                            rnntOptions]
_lib.rnnt_b200_lattice_align.restype = C.c_int
_lib.rnnt_b200_lattice_align.argtypes = [C.c_int, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P, rnntOptions]
_lib.get_workspace_size.restype = C.c_int
_lib.get_workspace_size.argtypes = [C.c_int, C.c_int, C.c_int, C.c_bool, C.POINTER(C.c_size_t), C.c_size_t]
_lib.get_warprnnt_version.restype = C.c_int
_lib.rnntGetStatusString.restype = C.c_char_p
_lib.rnntGetStatusString.argtypes = [C.c_int]
_lib.rnnt_b200_last_launch_count.restype = C.c_int
_lib.rnnt_b200_build_info.restype = C.c_char_p
_lib.rnnt_b200_set_profiling.restype = None
_lib.rnnt_b200_set_profiling.argtypes = [C.c_int]
_lib.rnnt_b200_last_kernel_ms.restype = C.c_int
_lib.rnnt_b200_last_kernel_ms.argtypes = [C.POINTER(C.c_float)]
_lib.rnnt_b200_profile_collect.restype = C.c_int
_lib.rnnt_b200_profile_collect.argtypes = [C.POINTER(C.c_float)]


def lib():
    """The loaded ctypes handle (tests and bench.py call the C-ABI through it)."""
    return _lib


def lib_path():
    return _LIB_PATH


def status_string(status):
    return _lib.rnntGetStatusString(int(status)).decode()


def workspace_size(maxT, maxU, minibatch, dtype_size=4, gpu=True):
    n = C.c_size_t(0)
    st = _lib.get_workspace_size(maxT, maxU, minibatch, gpu, C.byref(n), dtype_size)
    if st != RNNT_STATUS_SUCCESS:
        raise ValueError("get_workspace_size: " + status_string(st))
    return n.value


def last_launch_count():
    return _lib.rnnt_b200_last_launch_count()


def set_profiling(enabled):
    _lib.rnnt_b200_set_profiling(1 if enabled else 0)


def last_kernel_ms():
    """(rowstats, lattice, grad) milliseconds of the last profiled call on this thread."""
    out = (C.c_float * 3)()
    _lib.rnnt_b200_last_kernel_ms(out)
    return tuple(out)


def _options(acts, blank_label, num_threads=0):
    opt = rnntOptions()
    opt.loc = RNNT_GPU
    opt.num_threads = num_threads
    opt.stream = torch.cuda.current_stream(acts.device).cuda_stream
    opt.blank_label = blank_label
    opt.maxT = acts.size(1)
    opt.maxU = acts.size(2)
    opt.batch_first = True
    return opt


def _ptr(t):
    return t.data_ptr() if t is not None and t.numel() > 0 else None


_DUMMY_LABELS = {}   # device -> 1-element int32 tensor, kept alive for the life of the process


def _labels_ptr(labels):
    """U == 1 (no labels at all): the ABI still wants a non-null pointer.  The stand-in is a cached
    per-device tensor - a temporary would be freed before the (asynchronous) launch reads it."""
    if labels.numel() > 0:
        return labels.data_ptr()
    key = (labels.device.type, labels.device.index)
    if key not in _DUMMY_LABELS:
        _DUMMY_LABELS[key] = torch.zeros(1, dtype=torch.int32, device=labels.device)
    return _DUMMY_LABELS[key].data_ptr()


def require_same_device(ref, **tensors):
    """The async entry points dereference every pointer on `ref`'s device (host staging exists only in
    the synchronous C API), so a CPU or other-GPU tensor would be an illegal access, not an error."""
    for name, t in tensors.items():
        if t is not None and t.device != ref.device:
            raise RuntimeError("%s is on %s but the activations are on %s: all operator inputs must "
                               "live on the activations' CUDA device" % (name, t.device, ref.device))


def gpu_rnnt(acts, labels, input_lengths, label_lengths, costs, grads, blank_label, num_threads):
    """Reference signature (binding.cpp:84-91).  `costs` is a CPU tensor [N] (as the reference
    binding requires) or a CUDA tensor; `grads` is like `acts`, or empty for loss only.
    Returns 0 on success, raises on a library error (the reference ignored the status)."""
    if not acts.is_cuda:
        raise RuntimeError("gpu_rnnt needs CUDA tensors")
    N, T, U, V = acts.shape
    if acts.dtype == torch.float32:
        fn, esz = _lib.compute_rnnt_loss, 4
    elif acts.dtype == torch.float64:
        fn, esz = _lib.compute_rnnt_loss_fp64, 8
    else:
        raise TypeError("unsupported data type %s" % acts.dtype)
    with torch.cuda.device(acts.device):
        ws = torch.empty(workspace_size(T, U, N, esz), dtype=torch.uint8, device=acts.device)
        st = fn(acts.data_ptr(), _ptr(grads), _labels_ptr(labels), label_lengths.data_ptr(),
                input_lengths.data_ptr(), V, N, costs.data_ptr(), ws.data_ptr(),
                _options(acts, blank_label, num_threads))
    if st != RNNT_STATUS_SUCCESS:
        raise RuntimeError("compute_rnnt_loss failed: " + status_string(st))
    return 0


_FLOAT32_MAX = 3.4028234663852886e38


def grad_options(fastemit_lambda=0.0, clamp=-1.0):
    """Checked rnntGradOptions for the *_ex entries, or None when both options are off (the plain entries
    then run).  fastemit_lambda: finite, >= 0 (0 = off).  clamp: > 0 clips each gradient element to
    [-clamp, clamp] before grad_scale and the upstream gradient are applied; <= 0 = off; not NaN."""
    lam, c = float(fastemit_lambda), float(clamp)
    if not (math.isfinite(lam) and 0.0 <= lam <= _FLOAT32_MAX):
        raise ValueError("fastemit_lambda must be finite and >= 0 (float32), got %r" % (fastemit_lambda,))
    if math.isnan(c):
        raise ValueError("clamp must not be NaN")
    if lam == 0.0 and not c > 0.0:
        return None
    return rnntGradOptions(lam, c)


def lattice_options(delay_penalty=0.0):
    """Checked rnntLatticeOptions for the *_lat entries, or None when the delay penalty is off (the entries without
    lattice options then run).  delay_penalty: finite and >= 0 (float32); 0 = off.  A negative value is an error
    here (k2 ignores it)."""
    lam = float(delay_penalty)
    if not (math.isfinite(lam) and 0.0 <= lam <= _FLOAT32_MAX):
        raise ValueError("delay_penalty must be finite and >= 0 (float32), got %r" % (delay_penalty,))
    return None if lam == 0.0 else rnntLatticeOptions(lam)


_RNNT_TYPES = {'regular': RNNT_B200_RNNT_REGULAR, 'modified': RNNT_B200_RNNT_MODIFIED}


def rnnt_type_code(rnnt_type):
    """The C-ABI's rnnt_type for k2's `rnnt_type` name: 'regular' (any number of labels per frame) or 'modified'
    (at most one symbol per frame, include/rnnt.h RNNT_B200_RNNT_MODIFIED).  Anything else raises ValueError,
    k2's 'constrained' included."""
    if rnnt_type == 'constrained':
        raise ValueError("rnnt_type='constrained' is not supported; use 'regular' or 'modified'")
    if not isinstance(rnnt_type, str) or rnnt_type not in _RNNT_TYPES:
        raise ValueError("rnnt_type must be 'regular' or 'modified', got %r" % (rnnt_type,))
    return _RNNT_TYPES[rnnt_type]


def _dtype_code(acts):
    code = {torch.float32: RNNT_B200_FP32, torch.float64: RNNT_B200_FP64, torch.bfloat16: RNNT_B200_BF16,
            torch.float16: RNNT_B200_FP16}.get(acts.dtype)
    if code is None:
        raise TypeError("unsupported data type %s" % acts.dtype)
    return code


def _ex_options(fastemit_lambda, clamp):
    """rnntGradOptions for the *_ex entries; zeroed (both off) they launch exactly the plain entries' kernels."""
    gopt = grad_options(fastemit_lambda, clamp)
    return rnntGradOptions() if gopt is None else gopt


def _workspace(acts, T, U, N, workspace):
    """`workspace` when it holds the bytes these extents need, else a new one on the activations' device."""
    need = workspace_size(T, U, N, 8 if acts.dtype == torch.float64 else 4)
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device=acts.device)
    return workspace


def _loss_async(layout, T, U, N, V, acts, labels, input_lengths, label_lengths, costs, grads, blank_label,
                grad_scale, workspace, fastemit_lambda, clamp, delay_penalty=0.0, rnnt_type='regular'):
    gopt = _ex_options(fastemit_lambda, clamp)
    lopt = lattice_options(delay_penalty)
    topo = rnnt_type_code(rnnt_type)
    code = _dtype_code(acts)
    if layout == RNNT_B200_LAYOUT_TUNV and code not in (RNNT_B200_FP32, RNNT_B200_FP64):
        raise TypeError("unsupported data type %s for the time-major layout" % acts.dtype)
    with torch.cuda.device(acts.device):
        workspace = _workspace(acts, T, U, N, workspace)
        opt = _options(acts, blank_label)
        opt.maxT, opt.maxU = T, U
        args = (code, layout, acts.data_ptr(), _ptr(grads), _labels_ptr(labels), label_lengths.data_ptr(),
                input_lengths.data_ptr(), V, N, costs.data_ptr(), grad_scale, gopt)
        if topo != RNNT_B200_RNNT_REGULAR:
            st = _lib.rnnt_b200_loss_async_topo(*args, lopt or rnntLatticeOptions(), topo, workspace.data_ptr(), opt)
        elif lopt is None:
            st = _lib.rnnt_b200_loss_async_ex(*args, workspace.data_ptr(), opt)
        else:
            st = _lib.rnnt_b200_loss_async_lat(*args, lopt, workspace.data_ptr(), opt)
    if st != RNNT_STATUS_SUCCESS:
        raise RuntimeError("rnnt_b200_loss_async_ex failed: " + status_string(st))
    return workspace


def gpu_rnnt_async(acts, labels, input_lengths, label_lengths, costs, grads, blank_label,
                   grad_scale=1.0, workspace=None, *, fastemit_lambda=0.0, clamp=-1.0, delay_penalty=0.0,
                   rnnt_type='regular'):
    """Extension: no host synchronisation, `costs` on the device, gradients pre-multiplied by
    `grad_scale`.  Returns the workspace tensor (keep it alive until the stream has run).
    fastemit_lambda / clamp: gradient options (see grad_options); the costs do not depend on them, and
    with FastEmit on the gradient is not the gradient of the costs.  delay_penalty: the lattice option (see
    lattice_options); it changes the costs and the gradient.  rnnt_type: the topology (see rnnt_type_code)."""
    N, T, U, V = acts.shape
    return _loss_async(RNNT_B200_LAYOUT_NTUV, T, U, N, V, acts, labels, input_lengths, label_lengths, costs, grads,
                       blank_label, grad_scale, workspace, fastemit_lambda, clamp, delay_penalty, rnnt_type)


def gpu_rnnt_async_tunv(acts, labels, input_lengths, label_lengths, costs, grads, blank_label,
                        grad_scale=1.0, workspace=None, *, fastemit_lambda=0.0, clamp=-1.0, delay_penalty=0.0,
                        rnnt_type='regular'):
    """Time-major extension: `acts` / `grads` are [T, U, N, V] (the layout the reference's CPU path
    indexes for batch_first == false, cpu_rnnt.h:139-144); labels [N, U-1], lengths and costs [N].
    fp32 / fp64, no host synchronisation.  Returns the workspace tensor.  Gradient and lattice options and the
    topology as gpu_rnnt_async."""
    T, U, N, V = acts.shape
    return _loss_async(RNNT_B200_LAYOUT_TUNV, T, U, N, V, acts, labels, input_lengths, label_lengths, costs, grads,
                       blank_label, grad_scale, workspace, fastemit_lambda, clamp, delay_penalty, rnnt_type)


def _code16(acts):
    return {torch.bfloat16: RNNT_B200_BF16, torch.float16: RNNT_B200_FP16}.get(acts.dtype)


def costs_dtype(acts):
    """dtype of the per-utterance costs for a given activation dtype (fp32 for 16-bit storage)."""
    return torch.float32 if _code16(acts) else acts.dtype


def gpu_rnnt_forward(acts, labels, input_lengths, label_lengths, costs, blank_label,
                     prepare_backward=True, workspace=None, *, delay_penalty=0.0, rnnt_type='regular'):
    """Training-step split, first half: statistics + lattices into `workspace`, costs on the
    device, no synchronisation.  Returns the workspace tensor (hand it to gpu_rnnt_backward, with the same
    delay_penalty and rnnt_type)."""
    N, T, U, V = acts.shape
    lopt = lattice_options(delay_penalty)
    topo = rnnt_type_code(rnnt_type)
    code = _code16(acts)
    fn = {torch.float32: _lib.rnnt_b200_forward, torch.float64: _lib.rnnt_b200_forward_fp64}.get(acts.dtype)
    if code is None and fn is None:
        raise TypeError("unsupported data type %s" % acts.dtype)
    with torch.cuda.device(acts.device):
        workspace = _workspace(acts, T, U, N, workspace)
        args = (acts.data_ptr(), _labels_ptr(labels), label_lengths.data_ptr(), input_lengths.data_ptr(),
                V, N, costs.data_ptr(), 1 if prepare_backward else 0)
        tail = (workspace.data_ptr(), _options(acts, blank_label))
        if topo != RNNT_B200_RNNT_REGULAR:
            st = _lib.rnnt_b200_forward_topo(_dtype_code(acts), *args, lopt or rnntLatticeOptions(), topo, *tail)
        elif lopt is not None:
            st = _lib.rnnt_b200_forward_lat(_dtype_code(acts), *args, lopt, *tail)
        else:
            st = _lib.rnnt_b200_forward_16(code, *args, *tail) if code else fn(*args, *tail)
    if st != RNNT_STATUS_SUCCESS:
        raise RuntimeError("rnnt_b200_forward failed: " + status_string(st))
    return workspace


def gpu_rnnt_backward(acts, labels, input_lengths, label_lengths, grads, grad_costs, blank_label,
                      grad_scale, workspace, *, fastemit_lambda=0.0, clamp=-1.0, delay_penalty=0.0,
                      rnnt_type='regular'):
    """Second half: grads[b] = grad_scale * grad_costs[b] * d cost[b] / d acts[b] from the lattices
    gpu_rnnt_forward left in `workspace` (grad_costs: device tensor [N] or None for ones).
    With gradient options (see grad_options): grad_scale * grad_costs[b] * clip(g[b]), g[b] the FastEmit
    gradient when fastemit_lambda > 0.  delay_penalty and rnnt_type: the ones the forward half got."""
    N, T, U, V = acts.shape
    gopt = _ex_options(fastemit_lambda, clamp)
    lopt = lattice_options(delay_penalty)
    topo = rnnt_type_code(rnnt_type)
    code = _dtype_code(acts)
    with torch.cuda.device(acts.device):
        args = (code, acts.data_ptr(), grads.data_ptr(), _labels_ptr(labels), label_lengths.data_ptr(),
                input_lengths.data_ptr(), V, N, _ptr(grad_costs), grad_scale, gopt)
        tail = (workspace.data_ptr(), _options(acts, blank_label))
        if topo != RNNT_B200_RNNT_REGULAR:
            st = _lib.rnnt_b200_backward_topo(*args, lopt or rnntLatticeOptions(), topo, *tail)
        elif lopt is None:
            st = _lib.rnnt_b200_backward_ex(*args, *tail)
        else:
            st = _lib.rnnt_b200_backward_lat(*args, lopt, *tail)
    if st != RNNT_STATUS_SUCCESS:
        raise RuntimeError("rnnt_b200_backward_ex failed: " + status_string(st))
    return 0


def gpu_rnnt_align(acts, labels, input_lengths, label_lengths, frames, scores, blank_label, workspace=None, *,
                   rnnt_type='regular', time_major=False):
    """Forced alignment (include/rnnt.h rnnt_b200_align): the best path of each utterance's lattice.  Writes
    frames [N, U-1] int32 (the frame of each label, -1 past label_lengths and without a path) and scores [N]
    (its natural-log probability; costs_dtype(acts)), on the device, without synchronising.  acts: [N, T, U, V], or
    [T, U, N, V] with time_major (fp32 / fp64).  Returns the workspace tensor."""
    topo = rnnt_type_code(rnnt_type)
    code = _dtype_code(acts)
    layout = RNNT_B200_LAYOUT_TUNV if time_major else RNNT_B200_LAYOUT_NTUV
    if time_major:
        T, U, N, V = acts.shape
        if code not in (RNNT_B200_FP32, RNNT_B200_FP64):
            raise TypeError("unsupported data type %s for the time-major layout" % acts.dtype)
    else:
        N, T, U, V = acts.shape
    with torch.cuda.device(acts.device):
        workspace = _workspace(acts, T, U, N, workspace)
        opt = _options(acts, blank_label)
        opt.maxT, opt.maxU = T, U
        st = _lib.rnnt_b200_align(code, layout, acts.data_ptr(), _labels_ptr(labels), label_lengths.data_ptr(),
                                  input_lengths.data_ptr(), V, N, topo, _ptr(frames), scores.data_ptr(),
                                  workspace.data_ptr(), opt)
    if st != RNNT_STATUS_SUCCESS:
        raise RuntimeError("rnnt_b200_align failed: " + status_string(st))
    return workspace


def gpu_pruned_rnnt_align(logits, ranges, labels, input_lengths, label_lengths, frames, scores, blank_label,
                          workspace=None, *, rnnt_type='regular'):
    """gpu_rnnt_align for pruned logits [N, T, R, V] over the windows `ranges` [N, T] (include/rnnt.h
    rnnt_b200_pruned_align); the lattice is [T, labels.shape[1] + 1].  Returns the workspace tensor."""
    from .pruned import pruned_workspace_size
    topo = rnnt_type_code(rnnt_type)
    code = _dtype_code(logits)
    N, T, R, V = logits.shape
    U = labels.shape[1] + 1
    with torch.cuda.device(logits.device):
        need = pruned_workspace_size(T, U, R, N, 8 if logits.dtype == torch.float64 else 4)
        if workspace is None or workspace.numel() < need:
            workspace = torch.empty(need, dtype=torch.uint8, device=logits.device)
        opt = _options(logits, blank_label)
        opt.maxT, opt.maxU = T, U
        st = _lib.rnnt_b200_pruned_align(code, logits.data_ptr(), ranges.data_ptr(), R, _labels_ptr(labels),
                                         label_lengths.data_ptr(), input_lengths.data_ptr(), V, N, topo,
                                         _ptr(frames), scores.data_ptr(), workspace.data_ptr(), opt)
    if st != RNNT_STATUS_SUCCESS:
        raise RuntimeError("rnnt_b200_pruned_align failed: " + status_string(st))
    return workspace


def lattice_workspace_size(maxT, maxU, minibatch, dtype_size=4):
    """Bytes of workspace the lattice entries (include/rnnt.h rnnt_b200_lattice_forward) need."""
    n = C.c_size_t(0)
    st = _lib.rnnt_b200_lattice_workspace_size(maxT, maxU, minibatch, dtype_size, C.byref(n))
    if st != RNNT_STATUS_SUCCESS:
        raise RuntimeError("rnnt_b200_lattice_workspace_size failed: " + status_string(st))
    return n.value


def _lattice_options(py):
    """rnntOptions of a lattice call: extents from py [N, S+1, T], the current stream of py's device."""
    opt = rnntOptions()
    opt.loc = RNNT_GPU
    opt.stream = torch.cuda.current_stream(py.device).cuda_stream
    opt.maxU, opt.maxT = py.size(1), py.size(2)
    opt.batch_first = True
    return opt


def gpu_lattice_forward(px, py, input_lengths, label_lengths, costs, prepare_backward=True, workspace=None, *,
                        rnnt_type='regular'):
    """Loss on caller-supplied factors (include/rnnt.h rnnt_b200_lattice_forward): px [N, S, T] label and
    py [N, S+1, T] blank log-factors, contiguous, one storage type.  Writes costs [N] (costs_dtype(py)) on the device
    without synchronising; with prepare_backward the workspace also holds what gpu_lattice_backward reads.  Returns
    the workspace tensor."""
    topo = rnnt_type_code(rnnt_type)
    code = _dtype_code(py)
    N, U, T = py.shape
    with torch.cuda.device(py.device):
        need = lattice_workspace_size(T, U, N, 8 if py.dtype == torch.float64 else 4)
        if workspace is None or workspace.numel() < need:
            workspace = torch.empty(need, dtype=torch.uint8, device=py.device)
        st = _lib.rnnt_b200_lattice_forward(code, _ptr(px), py.data_ptr(), label_lengths.data_ptr(),
                                            input_lengths.data_ptr(), N, topo, costs.data_ptr(),
                                            1 if prepare_backward else 0, workspace.data_ptr(), _lattice_options(py))
    if st != RNNT_STATUS_SUCCESS:
        raise RuntimeError("rnnt_b200_lattice_forward failed: " + status_string(st))
    return workspace


def gpu_lattice_backward(px_grad, py_grad, input_lengths, label_lengths, grad_costs, grad_scale, workspace, *,
                         rnnt_type='regular'):
    """Second half: px_grad / py_grad (shaped and typed as px / py) = grad_scale * grad_costs[b] * d cost[b] / d
    px / py from the workspace gpu_lattice_forward(prepare_backward=True) filled, with the same rnnt_type.
    grad_costs: device tensor [N] in costs_dtype, or None for ones.  Every element is written."""
    topo = rnnt_type_code(rnnt_type)
    code = _dtype_code(py_grad)
    N = py_grad.size(0)
    with torch.cuda.device(py_grad.device):
        st = _lib.rnnt_b200_lattice_backward(code, _ptr(px_grad), py_grad.data_ptr(), label_lengths.data_ptr(),
                                             input_lengths.data_ptr(), N, topo, _ptr(grad_costs), grad_scale,
                                             workspace.data_ptr(), _lattice_options(py_grad))
    if st != RNNT_STATUS_SUCCESS:
        raise RuntimeError("rnnt_b200_lattice_backward failed: " + status_string(st))
    return 0


def gpu_lattice_align(px, py, input_lengths, label_lengths, frames, scores, workspace=None, *, rnnt_type='regular'):
    """Forced alignment on caller-supplied factors (include/rnnt.h rnnt_b200_lattice_align): frames [N, S] int32
    and scores [N] (costs_dtype(py)) as gpu_rnnt_align, on the device, without synchronising.  Returns the
    workspace tensor."""
    topo = rnnt_type_code(rnnt_type)
    code = _dtype_code(py)
    N, U, T = py.shape
    with torch.cuda.device(py.device):
        need = lattice_workspace_size(T, U, N, 8 if py.dtype == torch.float64 else 4)
        if workspace is None or workspace.numel() < need:
            workspace = torch.empty(need, dtype=torch.uint8, device=py.device)
        st = _lib.rnnt_b200_lattice_align(code, _ptr(px), py.data_ptr(), label_lengths.data_ptr(),
                                          input_lengths.data_ptr(), N, topo, _ptr(frames), scores.data_ptr(),
                                          workspace.data_ptr(), _lattice_options(py))
    if st != RNNT_STATUS_SUCCESS:
        raise RuntimeError("rnnt_b200_lattice_align failed: " + status_string(st))
    return workspace


_lib.rnnt_b200_debug_log_likelihoods.restype = C.c_int
_lib.rnnt_b200_debug_log_likelihoods.argtypes = [_P, C.c_int, C.c_int, C.c_int, C.c_size_t, _P, _P]


def read_log_likelihoods(workspace, maxT, maxU, minibatch, dtype_size=4):
    """(llForward, llBackward) of the last loss+gradient call that used `workspace` (test hook)."""
    import numpy as np
    f, b = np.zeros(minibatch), np.zeros(minibatch)
    st = _lib.rnnt_b200_debug_log_likelihoods(workspace.data_ptr(), maxT, maxU, minibatch, dtype_size,
                                              f.ctypes.data, b.ctypes.data)
    if st != RNNT_STATUS_SUCCESS:
        raise RuntimeError("rnnt_b200_debug_log_likelihoods: " + status_string(st))
    return f, b


def profile_collect():
    """(calls, (rowstats, lattice, grad) mean ms) over the profiled calls since the last collect."""
    out = (C.c_float * 3)()
    n = _lib.rnnt_b200_profile_collect(out)
    return n, tuple(out)


def cpu_rnnt(acts, labels, input_lengths, label_lengths, costs, grads, blank_label, num_threads):
    """Reference signature (binding.cpp:12-19).  Not available: the H100 build is the device
    path only and must not fall back to a host implementation."""
    raise RuntimeError("warprnnt_pytorch (H100 build): cpu_rnnt is not available - "
                       "move the tensors to a CUDA device")
