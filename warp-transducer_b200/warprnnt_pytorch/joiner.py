"""The RNN-T loss of a real joiner without the [N, T, U, V] logits (DESIGN.md §14).  icefall's ``Joiner``,
torchaudio's ``RNNTJoiner`` and NeMo's ``RNNTJoint`` compute

    logits[b, t, u, :] = weight @ act(enc[b, t] + pred[b, u]) + bias          act = tanh or relu

with enc [N, T, H] and pred [N, U, H] already projected to the joiner width H.  ``joiner_log_probs`` reduces that
joiner straight to the lattice factors of ``rnnt_lattice_loss`` on bf16 tensor cores, chunk by chunk, and its
backward runs the contraction in reverse, so neither the logits nor their gradient ever exist:

    px, py = joiner_log_probs(enc, pred, weight, bias, labels, act_lens, label_lens)   # px [N,S,T], py [N,S+1,T]
    loss = joiner_rnnt_loss(enc, pred, weight, bias, labels, act_lens, label_lens)
    frames, scores = rnnt_lattice_forced_align(*joiner_log_probs(...), act_lens, label_lens)

enc, pred, weight [V, H] (nn.Linear's layout) and bias [V] (or None) are bf16 CUDA tensors; pass a joiner's fp32
master weights as ``weight.to(torch.bfloat16)`` and autograd carries the gradient back to them.

The pruned step of pruned RNN-T (DESIGN.md §15) runs the same joiner on the windows of the pruning ranges only,
without the [N, T, R, V] logits of ``prune_joint_inputs`` -> joiner -> ``pruned_rnnt_loss``:

    simple, ranges = add_joint_rnnt_loss_with_ranges(am_proj, lm_proj, labels, act_lens, label_lens, s_range=5)
    pruned = pruned_joiner_rnnt_loss(enc, pred, weight, bias, labels, act_lens, label_lens, ranges, 5)

Both take NeMo's joint dropout, Sequential(act, Dropout(p), Linear), on the hidden activation (DESIGN.md §16), with
the mask regenerated in the backward from a 64-bit seed instead of stored:

    loss = joiner_rnnt_loss(enc, pred, weight, bias, labels, act_lens, label_lens, activation='relu', dropout=0.2)
"""
import ctypes as C

import torch
from torch.autograd import Function
from torch.nn import Module

from . import warp_rnnt
from ._checks import LengthCheck, check_contiguous, check_dim, check_type
from .lattice import rnnt_lattice_loss

_lib = warp_rnnt.lib()
_P = C.c_void_p
_lib.rnnt_b200_joiner_workspace_size.restype = C.c_int
_lib.rnnt_b200_joiner_workspace_size.argtypes = [C.c_int] * 6 + [C.POINTER(C.c_size_t)]
_lib.rnnt_b200_joiner_forward.restype = C.c_int
_lib.rnnt_b200_joiner_forward.argtypes = [C.c_int, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int,
                                          _P, _P, _P, warp_rnnt.rnntOptions]
_lib.rnnt_b200_joiner_backward.restype = C.c_int
_lib.rnnt_b200_joiner_backward.argtypes = [C.c_int, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int,
                                           _P, _P, _P, _P, _P, _P, _P, warp_rnnt.rnntOptions]
_lib.rnnt_b200_joiner_last_launch_count.restype = C.c_int
_lib.rnnt_b200_pruned_joiner_workspace_size.restype = C.c_int
_lib.rnnt_b200_pruned_joiner_workspace_size.argtypes = [C.c_int] * 7 + [C.POINTER(C.c_size_t)]
_lib.rnnt_b200_pruned_joiner_forward.restype = C.c_int
_lib.rnnt_b200_pruned_joiner_forward.argtypes = [C.c_int, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int,
                                                 C.c_int, C.c_int, _P, _P, _P, warp_rnnt.rnntOptions]
_lib.rnnt_b200_pruned_joiner_backward.restype = C.c_int
_lib.rnnt_b200_pruned_joiner_backward.argtypes = [C.c_int, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int,
                                                  C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P,
                                                  warp_rnnt.rnntOptions]


class rnntJoinerDropout(C.Structure):
    """include/rnnt.h struct rnntJoinerDropout, passed by value to the *_drop entries."""
    _fields_ = [("p", C.c_float), ("seed", C.c_void_p)]


def _drop_argtypes(plain):
    """The *_drop entry's arguments: the plain entry's with the dropout struct before the workspace."""
    return plain[:-2] + [rnntJoinerDropout] + plain[-2:]


for _name in ("joiner_forward", "joiner_backward", "pruned_joiner_forward", "pruned_joiner_backward"):
    _f = getattr(_lib, "rnnt_b200_%s_drop" % _name)
    _f.restype = C.c_int
    _f.argtypes = _drop_argtypes(getattr(_lib, "rnnt_b200_" + _name).argtypes)

RNNT_B200_ACT_TANH, RNNT_B200_ACT_RELU = 0, 1
_ACTIVATIONS = {'tanh': RNNT_B200_ACT_TANH, 'relu': RNNT_B200_ACT_RELU}


def activation_code(activation):
    """The C-ABI's activation code for 'tanh' or 'relu'; ValueError otherwise."""
    if activation not in _ACTIVATIONS:
        raise ValueError("activation must be 'tanh' or 'relu', got %r" % (activation,))
    return _ACTIVATIONS[activation]


def _chunk(chunk_cells):
    if chunk_cells is None:
        return 0
    if isinstance(chunk_cells, bool) or not isinstance(chunk_cells, int) or not 1 <= chunk_cells < 2 ** 31:
        raise ValueError("chunk_cells must be None or an int in [1, 2^31), got %r" % (chunk_cells,))
    return chunk_cells


def dropout_p(dropout):
    """The dropout probability as the C-ABI takes it (a float32 in [0, 1)); ValueError otherwise, a bool included."""
    if isinstance(dropout, bool) or not isinstance(dropout, (int, float)):
        raise ValueError("dropout must be a float in [0, 1), got %r" % (dropout,))
    p = float(dropout)
    if not (0.0 <= p < 1.0) or C.c_float(p).value >= 1.0:
        raise ValueError("dropout must be a float in [0, 1), got %r" % (dropout,))
    return p


def _check_seed(seed):
    """An explicit dropout seed: an int64 tensor of one element (the device is checked with the inputs')."""
    if seed is None:
        return
    if not isinstance(seed, torch.Tensor) or seed.dtype is not torch.int64:
        raise TypeError("dropout_seed must be None or an int64 tensor of one element, got %s"
                        % (seed.dtype if isinstance(seed, torch.Tensor) else type(seed).__name__))
    if seed.numel() != 1:
        raise ValueError("dropout_seed must have one element, got shape %s" % (tuple(seed.shape),))


def _seed_on(seed, device):
    """The seed tensor a dropout call reads on the device: a fresh one from torch's CUDA generator when None (no host
    synchronisation; torch.manual_seed reproduces it), else the caller's, which must be on the inputs' device."""
    if seed is None:
        return torch.empty(1, dtype=torch.int64, device=device).random_()
    if not seed.is_cuda or seed.device != device:
        raise RuntimeError("dropout_seed must be on the inputs' device %s, got %s" % (device, seed.device))
    return seed.reshape(1).contiguous()


def workspace_size(maxT, maxU, minibatch, hidden, alphabet_size, chunk_cells=None, s_range=None):
    """Bytes of the joiner's workspace (include/rnnt.h rnnt_b200_joiner_workspace_size), or with s_range of the
    pruned joiner's (rnnt_b200_pruned_joiner_workspace_size)."""
    n = C.c_size_t(0)
    if s_range is None:
        name = "rnnt_b200_joiner_workspace_size"
        st = _lib.rnnt_b200_joiner_workspace_size(maxT, maxU, minibatch, hidden, alphabet_size, _chunk(chunk_cells),
                                                  C.byref(n))
    else:
        name = "rnnt_b200_pruned_joiner_workspace_size"
        st = _lib.rnnt_b200_pruned_joiner_workspace_size(maxT, maxU, s_range, minibatch, hidden, alphabet_size,
                                                         _chunk(chunk_cells), C.byref(n))
    if st != warp_rnnt.RNNT_STATUS_SUCCESS:
        raise ValueError(name + ": " + warp_rnnt.status_string(st))
    return n.value


def last_launch_count():
    """Kernels the last joiner call on this thread launched."""
    return _lib.rnnt_b200_joiner_last_launch_count()


def _check_window(ranges, s_range, N, T):
    """pruned_rnnt_loss's rules for ranges (int32 [N, T], contiguous) and a positive int s_range, N T R < 2^31.  A
    pruned call always has its window: ranges=None is a TypeError, never the dense joiner."""
    if not isinstance(ranges, torch.Tensor):
        raise TypeError("ranges must be an int32 tensor [N, T], got %s" % type(ranges).__name__)
    if isinstance(s_range, bool) or not isinstance(s_range, int) or s_range < 1:
        raise ValueError("s_range must be a positive int, got %r" % (s_range,))
    check_type(ranges, torch.int32, "ranges")
    check_contiguous(ranges, "ranges")
    check_dim(ranges, 2, "ranges")
    if tuple(ranges.shape) != (N, T):
        raise ValueError("ranges must be [N, T] = [%d, %d], got %s" % (N, T, tuple(ranges.shape)))
    if N * T * s_range >= 2 ** 31:
        raise ValueError("N * T * s_range must be below 2^31, got %d" % (N * T * s_range))


def _check_inputs(enc, pred, weight, bias, labels, act_lens, label_lens, blank, activation, chunk_cells,
                  window=None):
    """rnnt_loss's rules and exception types: ValueError for an option, a rank, a shape, an extent or a
    non-contiguous tensor, TypeError for a dtype, RuntimeError for a CPU tensor or a second device.  With a window
    (ranges, s_range), a pruned call, pruned_rnnt_loss's rules for it too.  Returns the deferred T == max(act_lens),
    S == max(label_lens) check."""
    activation_code(activation)
    _chunk(chunk_cells)
    for name, t in (("enc", enc), ("pred", pred), ("weight", weight), ("bias", bias)):
        if t is not None and t.dtype is not torch.bfloat16:
            raise TypeError("%s must be torch.bfloat16 (fp16 and fp32 are not supported), got %s" % (name, t.dtype))
    check_type(labels, torch.int32, "labels")
    check_type(act_lens, torch.int32, "lengths")
    check_type(label_lens, torch.int32, "label_lengths")
    for name, t, rank in (("enc", enc, 3), ("pred", pred, 3), ("weight", weight, 2), ("bias", bias, 1),
                          ("labels", labels, 2), ("lengths", act_lens, 1), ("label_lengths", label_lens, 1)):
        if t is not None:
            check_contiguous(t, name)
            check_dim(t, rank, name)
    N, T, H = enc.shape
    U = pred.shape[1]
    V = weight.shape[0]
    if pred.shape[0] != N or pred.shape[2] != H:
        raise ValueError("pred must be [N, U, H] = [%d, U, %d], got %s" % (N, H, list(pred.shape)))
    if weight.shape[1] != H:
        raise ValueError("weight must be [V, H] with H = %d, got %s" % (H, list(weight.shape)))
    if bias is not None and bias.shape[0] != V:
        raise ValueError("bias must be [V] = [%d], got %s" % (V, list(bias.shape)))
    if tuple(labels.shape) != (N, U - 1):
        raise ValueError("labels must be [N, U-1] = %s, got %s" % ([N, U - 1], list(labels.shape)))
    if act_lens.shape[0] != N:
        raise ValueError("must have a length per example.")
    if label_lens.shape[0] != N:
        raise ValueError("must have a label length per example.")
    if H % 16 != 0 or not 16 <= H <= 1024:
        raise ValueError("the joiner width H must be a multiple of 16 in [16, 1024], got %d" % H)
    if V < 2:
        raise ValueError("the alphabet must have at least 2 symbols, got %d" % V)
    if not 0 <= blank < V:
        raise ValueError("blank must be in [0, %d), got %d" % (V, blank))
    if N < 1 or T < 1 or U < 1:
        raise ValueError("enc and pred must have at least one utterance, frame and context")
    if U > 1024:
        raise ValueError("U must be at most 1024, got %d" % U)
    if N * T * U >= 2 ** 31:
        raise ValueError("N * T * U must be below 2^31, got %d" % (N * T * U))
    tensors = dict(pred=pred, weight=weight, bias=bias, labels=labels, act_lens=act_lens, label_lens=label_lens)
    if window is not None:
        _check_window(*window, N, T)
        tensors["ranges"] = window[0]
    if not all(t.is_cuda for t in [enc] + [t for t in tensors.values() if t is not None]):
        raise RuntimeError("warprnnt_pytorch (H100 build) runs on CUDA tensors only; there is no CPU fallback")
    warp_rnnt.require_same_device(enc, **tensors)
    return LengthCheck(act_lens, label_lens, T, U)


def _options(enc, U, blank):
    opt = warp_rnnt.rnntOptions()
    opt.loc = warp_rnnt.RNNT_GPU
    opt.stream = torch.cuda.current_stream(enc.device).cuda_stream
    opt.blank_label = blank
    opt.maxT = enc.size(1)
    opt.maxU = U
    return opt


def _ptr(t):
    return t.data_ptr() if t is not None and t.numel() > 0 else None


def _inputs(enc, pred, weight, bias, labels, act_lens, label_lens, ranges, s_range):
    """The entry's name and its leading arguments (the window follows the lengths on the pruned entries).  Either
    of ranges and s_range makes the call pruned, and a pruned call needs both."""
    head = [enc.data_ptr(), pred.data_ptr(), weight.data_ptr(), _ptr(bias), _ptr(labels), label_lens.data_ptr(),
            act_lens.data_ptr()]
    if ranges is None and s_range is None:
        return "rnnt_b200_joiner", head
    if ranges is None or s_range is None:
        raise ValueError("a pruned joiner call needs both ranges and s_range")
    return "rnnt_b200_pruned_joiner", head + [ranges.data_ptr(), s_range]


def _drop(name, dropout, seed):
    """The entry (plain, or its *_drop form when dropout > 0) and the trailing dropout argument, if any."""
    if not dropout:
        return getattr(_lib, name), []
    if seed is None:
        raise ValueError("a dropout call needs its seed tensor")
    return getattr(_lib, name + "_drop"), [rnntJoinerDropout(dropout, seed.data_ptr())]


def gpu_joiner_forward(enc, pred, weight, bias, labels, act_lens, label_lens, px, py, blank, activation,
                       chunk_cells=None, workspace=None, ranges=None, s_range=None, dropout=0.0, seed=None):
    """px [N, S, T] and py [N, S+1, T] (float32, every element written) from the joiner's inputs, checked by the
    caller (include/rnnt.h rnnt_b200_joiner_forward; with ranges and s_range, rnnt_b200_pruned_joiner_forward; with
    dropout > 0 their *_drop forms, reading the int64 seed tensor on the device).  Returns the workspace, which the
    backward reads."""
    N, T, H = enc.shape
    U, V = pred.shape[1], weight.shape[0]
    name, head = _inputs(enc, pred, weight, bias, labels, act_lens, label_lens, ranges, s_range)
    fn, drop = _drop(name + "_forward", dropout, seed)
    with torch.cuda.device(enc.device):
        need = workspace_size(T, U, N, H, V, chunk_cells, s_range)
        if workspace is None or workspace.numel() < need:
            workspace = torch.empty(need, dtype=torch.uint8, device=enc.device)
        st = fn(activation_code(activation), *head, H, V, N, _chunk(chunk_cells), _ptr(px), py.data_ptr(), *drop,
                workspace.data_ptr(), _options(enc, U, blank))
    if st != warp_rnnt.RNNT_STATUS_SUCCESS:
        raise RuntimeError(name + "_forward failed: " + warp_rnnt.status_string(st))
    return workspace


def gpu_joiner_backward(enc, pred, weight, bias, labels, act_lens, label_lens, dpx, dpy, grad_enc, grad_pred,
                        grad_weight, grad_bias, blank, activation, chunk_cells, workspace, ranges=None,
                        s_range=None, dropout=0.0, seed=None):
    """The four bf16 gradients from dpx, dpy (float32, shaped as px, py) and the workspace of gpu_joiner_forward
    with the same arguments, dropout and seed included (include/rnnt.h rnnt_b200_joiner_backward /
    rnnt_b200_pruned_joiner_backward, or their *_drop forms)."""
    N, T, H = enc.shape
    U, V = pred.shape[1], weight.shape[0]
    name, head = _inputs(enc, pred, weight, bias, labels, act_lens, label_lens, ranges, s_range)
    fn, drop = _drop(name + "_backward", dropout, seed)
    with torch.cuda.device(enc.device):
        st = fn(activation_code(activation), *head, H, V, N, _chunk(chunk_cells), _ptr(dpx), dpy.data_ptr(),
                grad_enc.data_ptr(), grad_pred.data_ptr(), grad_weight.data_ptr(), _ptr(grad_bias), *drop,
                workspace.data_ptr(), _options(enc, U, blank))
    if st != warp_rnnt.RNNT_STATUS_SUCCESS:
        raise RuntimeError(name + "_backward failed: " + warp_rnnt.status_string(st))


class _JoinerLogProbs(Function):
    """The dense joiner (window None), or with a window (ranges, s_range) the pruned one; dropout > 0 on h with the
    seed tensor (None: drawn from torch's CUDA generator).  forward: 2 launches per chunk (the pruned call 1 more,
    the -inf fill), px / py and the per-row lse.  backward: 5 launches per chunk and 1 more, from the lse the forward
    left in the workspace and the same seed."""

    @staticmethod
    def forward(ctx, enc, pred, weight, bias, labels, act_lens, label_lens, blank, activation, chunk_cells,
                window=None, dropout=0.0, seed=None):
        dropout = dropout_p(dropout)
        _check_seed(seed)
        length_check = _check_inputs(enc, pred, weight, bias, labels, act_lens, label_lens, blank, activation,
                                     chunk_cells, window)
        seed = _seed_on(seed, enc.device) if dropout else None
        ranges, s_range = window if window is not None else (None, None)
        N, T, _ = enc.shape
        S = pred.shape[1] - 1
        px = torch.empty((N, S, T), dtype=torch.float32, device=enc.device)
        py = torch.empty((N, S + 1, T), dtype=torch.float32, device=enc.device)
        ws = gpu_joiner_forward(enc, pred, weight, bias, labels, act_lens, label_lens, px, py, blank, activation,
                                chunk_cells, ranges=ranges, s_range=s_range, dropout=dropout, seed=seed)
        length_check.finish()
        ctx.save_for_backward(enc, pred, weight, bias, labels, act_lens, label_lens, ranges, seed)
        ctx.workspace = ws
        ctx.args = (blank, activation, chunk_cells, s_range, dropout)
        return px, py

    @staticmethod
    def backward(ctx, dpx, dpy):
        enc, pred, weight, bias, labels, act_lens, label_lens, ranges, seed = ctx.saved_tensors
        blank, activation, chunk_cells, s_range, dropout = ctx.args
        N, T, _ = enc.shape
        S = pred.shape[1] - 1
        dpx = (torch.zeros((N, S, T), dtype=torch.float32, device=enc.device) if dpx is None
               else dpx.to(torch.float32).contiguous())
        dpy = (torch.zeros((N, S + 1, T), dtype=torch.float32, device=enc.device) if dpy is None
               else dpy.to(torch.float32).contiguous())
        grad_enc, grad_pred, grad_weight = torch.empty_like(enc), torch.empty_like(pred), torch.empty_like(weight)
        grad_bias = torch.empty_like(bias) if bias is not None else None
        gpu_joiner_backward(enc, pred, weight, bias, labels, act_lens, label_lens, dpx, dpy, grad_enc, grad_pred,
                            grad_weight, grad_bias, blank, activation, chunk_cells, ctx.workspace, ranges, s_range,
                            dropout, seed)
        need = ctx.needs_input_grad
        return (grad_enc if need[0] else None, grad_pred if need[1] else None, grad_weight if need[2] else None,
                grad_bias if bias is not None and need[3] else None, None, None, None, None, None, None, None, None,
                None)


def joiner_log_probs(enc, pred, weight, bias, labels, act_lens, label_lens, blank=0, *, activation='tanh',
                     chunk_cells=None, dropout=0.0, dropout_seed=None):
    """The lattice factors of the joiner  logits = weight act(enc[b,t] + pred[b,u]) + bias,  without the logits.

    enc [N, T, H], pred [N, U, H], weight [V, H], bias [V] or None: bf16, contiguous, on one CUDA device, with
    H % 16 == 0, 16 <= H <= 1024, V >= 2, U <= 1024 and N T U < 2^31.  labels [N, U-1], act_lens and label_lens [N]
    are int32, with T == max(act_lens) and U == max(label_lens) + 1 (checked after the kernels are queued).

    Returns float32 px [N, U-1, T] (label s at frame t) and py [N, U, T] (blank at (t, s)), rnnt_lattice_loss's
    orientation: px[b,s,t] = logit_{labels[b,s]} - lse and py[b,s,t] = logit_blank - lse, -inf on padding.  The
    hidden activation is h = round_bf16(act(fp32(enc) + fp32(pred))) with act tanhf or relu: one rounding fewer than
    a bf16 eager joiner, which also rounds the sum.  The logits are h weight^T + bias in fp32 and lse their fp32
    logsumexp.  A label outside [0, V) gives px = NaN on its row.  Both outputs are differentiable: the
    backward returns bf16 gradients of enc, pred, weight and bias, accumulated in fp32 and bitwise deterministic for
    a given chunk_cells.

    chunk_cells: cells per pass through the scratch; None keeps the scratch within 256 MiB.

    dropout = p in [0, 1): NeMo's joint dropout on h (DESIGN.md §16).  The logits use h~ = keep ? round_bf16(h / (1 -
    p)) : 0, the backward the same mask (regenerated, not stored) and act' from the undropped h.  Element k of cell
    (b, t, u) is dropped iff word k & 3 of Philox4x32-10(ctr (k >> 2, (b U + u) T + t, 0, 0), key = the seed's two
    halves) is below floor(p 2^32): the mask depends on the padded extents T and U, as eager dropout on [N, T, U, H]
    does, and never on chunk_cells.  dropout_seed: None draws one int64 seed on the inputs' device from torch's CUDA
    generator (no host sync; torch.manual_seed, CUDA-graph replays and torch.utils.checkpoint behave as for
    nn.Dropout); or an int64 CUDA tensor of one element on that device.  dropout=0 is exactly the call without it."""
    return _JoinerLogProbs.apply(enc, pred, weight, bias, labels, act_lens, label_lens, blank, activation,
                                 chunk_cells, None, dropout, dropout_seed)


def pruned_joiner_log_probs(enc, pred, weight, bias, labels, act_lens, label_lens, ranges, s_range, blank=0, *,
                            activation='tanh', chunk_cells=None, dropout=0.0, dropout_seed=None):
    """joiner_log_probs on the pruned lattice of pruned_rnnt_loss, without the [N, T, R, V] logits (DESIGN.md §15).

    ranges [N, T] int32 (contiguous, on the inputs' device) and s_range = R, a positive int: row (b, t, r), r < R,
    stands for cell (t, ranges[b, t] + r), and is padding unless t < T_b and 0 <= ranges[b, t] + r <= S_b (any int32
    start is allowed, and R > U).  Returns px [N, U-1, T] and py [N, U, T] as joiner_log_probs does: its values on
    the cells a valid row covers, -inf everywhere else; dpx / dpy are read only on those cells.  The other arguments
    and the gradients are joiner_log_probs's; chunk_cells counts rows (b, t, r).  With s_range = U and ranges == 0
    both the factors and the gradients are bitwise joiner_log_probs's.  The alignment of the pruned lattice is
    rnnt_lattice_forced_align(*pruned_joiner_log_probs(...), act_lens, label_lens).  dropout and dropout_seed are
    joiner_log_probs's; a row uses the mask of the cell it stands for, so with the same seed the result is the dense
    one's on the covered cells."""
    return _JoinerLogProbs.apply(enc, pred, weight, bias, labels, act_lens, label_lens, blank, activation,
                                 chunk_cells, (ranges, s_range), dropout, dropout_seed)


def _delay(px, act_lens, delay_penalty):
    """px + delay_penalty ((T_b - 1) / 2 - t): rnnt_loss's delay-penalised label factors."""
    T = px.shape[2]
    t = torch.arange(T, device=px.device, dtype=torch.float32)
    tb = act_lens.to(torch.float32).clamp(1, T).unsqueeze(1)
    return px + (delay_penalty * ((tb - 1) * 0.5 - t)).unsqueeze(1)


def joiner_rnnt_loss(enc, pred, weight, bias, labels, act_lens, label_lens, blank=0, reduction='mean', *,
                     activation='tanh', rnnt_type='regular', delay_penalty=0.0, dropout=0.0, dropout_seed=None):
    """RNN-T loss of the joiner  logits = weight act(enc[b,t] + pred[b,u]) + bias  (see joiner_log_probs), without
    the [N, T, U, V] logits or their gradient:

        rnnt_lattice_loss(px + delay_penalty ((T_b - 1)/2 - t), py, act_lens, label_lens, reduction, rnnt_type)

    on (px, py) = joiner_log_probs(...).  reduction, rnnt_type and delay_penalty are rnnt_loss's; dropout and
    dropout_seed are joiner_log_probs's (applied whenever dropout > 0: the module form applies it in training only)."""
    return _loss(enc, pred, weight, bias, labels, act_lens, label_lens, blank, reduction, activation, rnnt_type,
                 delay_penalty, None, dropout, dropout_seed)


def pruned_joiner_rnnt_loss(enc, pred, weight, bias, labels, act_lens, label_lens, ranges, s_range, blank=0,
                            reduction='mean', *, activation='tanh', rnnt_type='regular', delay_penalty=0.0,
                            dropout=0.0, dropout_seed=None):
    """Pruned RNN-T loss of the joiner  logits = weight act(enc[b,t] + pred[b,u]) + bias  on the windows
    (ranges, s_range) of add_joint_rnnt_loss_with_ranges, without the [N, T, R, V] logits or their gradient: what
    prune_joint_inputs -> joiner -> pruned_rnnt_loss computes, as

        rnnt_lattice_loss(px + delay_penalty ((T_b - 1)/2 - t), py, act_lens, label_lens, reduction, rnnt_type)

    on (px, py) = pruned_joiner_log_probs(...).  An utterance whose windows leave no path costs +inf with zero
    gradients.  reduction, rnnt_type and delay_penalty are pruned_rnnt_loss's; dropout and dropout_seed are
    joiner_log_probs's."""
    return _loss(enc, pred, weight, bias, labels, act_lens, label_lens, blank, reduction, activation, rnnt_type,
                 delay_penalty, (ranges, s_range), dropout, dropout_seed)


def _loss(enc, pred, weight, bias, labels, act_lens, label_lens, blank, reduction, activation, rnnt_type,
          delay_penalty, window=None, dropout=0.0, dropout_seed=None):
    warp_rnnt.rnnt_type_code(rnnt_type)
    warp_rnnt.lattice_options(delay_penalty)
    if reduction not in ('none', 'sum', 'mean'):
        raise ValueError("reduction must be 'none', 'sum' or 'mean'")
    px, py = _JoinerLogProbs.apply(enc, pred, weight, bias, labels, act_lens, label_lens, blank, activation, None,
                                   window, dropout, dropout_seed)
    if delay_penalty:
        px = _delay(px, act_lens, float(delay_penalty))
    return rnnt_lattice_loss(px, py, act_lens, label_lens, reduction, rnnt_type=rnnt_type)


class JoinerRNNTLoss(Module):
    """Module form of joiner_rnnt_loss: JoinerRNNTLoss(blank=0, reduction='mean', *, activation='tanh',
    rnnt_type='regular', delay_penalty=0.0, dropout=0.0); forward(enc, pred, weight, bias, labels, act_lens,
    label_lens).  dropout applies in training mode only, as nn.Dropout's, with a fresh seed per call."""

    def __init__(self, blank=0, reduction='mean', *, activation='tanh', rnnt_type='regular', delay_penalty=0.0,
                 dropout=0.0):
        super().__init__()
        activation_code(activation)
        warp_rnnt.rnnt_type_code(rnnt_type)
        warp_rnnt.lattice_options(delay_penalty)
        if reduction not in ('none', 'sum', 'mean'):
            raise ValueError("reduction must be 'none', 'sum' or 'mean'")
        self.blank, self.reduction = blank, reduction
        self.activation, self.rnnt_type, self.delay_penalty = activation, rnnt_type, delay_penalty
        self.dropout = dropout_p(dropout)

    def forward(self, enc, pred, weight, bias, labels, act_lens, label_lens):
        return joiner_rnnt_loss(enc, pred, weight, bias, labels, act_lens, label_lens, self.blank, self.reduction,
                                activation=self.activation, rnnt_type=self.rnnt_type,
                                delay_penalty=self.delay_penalty, dropout=self.dropout if self.training else 0.0)


class PrunedJoinerRNNTLoss(Module):
    """Module form of pruned_joiner_rnnt_loss: PrunedJoinerRNNTLoss(blank=0, reduction='mean', *, activation='tanh',
    rnnt_type='regular', delay_penalty=0.0, dropout=0.0); forward(enc, pred, weight, bias, labels, act_lens,
    label_lens, ranges, s_range).  dropout applies in training mode only, as nn.Dropout's."""

    def __init__(self, blank=0, reduction='mean', *, activation='tanh', rnnt_type='regular', delay_penalty=0.0,
                 dropout=0.0):
        super().__init__()
        activation_code(activation)
        warp_rnnt.rnnt_type_code(rnnt_type)
        warp_rnnt.lattice_options(delay_penalty)
        if reduction not in ('none', 'sum', 'mean'):
            raise ValueError("reduction must be 'none', 'sum' or 'mean'")
        self.blank, self.reduction = blank, reduction
        self.activation, self.rnnt_type, self.delay_penalty = activation, rnnt_type, delay_penalty
        self.dropout = dropout_p(dropout)

    def forward(self, enc, pred, weight, bias, labels, act_lens, label_lens, ranges, s_range):
        return pruned_joiner_rnnt_loss(enc, pred, weight, bias, labels, act_lens, label_lens, ranges, s_range,
                                       self.blank, self.reduction, activation=self.activation,
                                       rnnt_type=self.rnnt_type, delay_penalty=self.delay_penalty,
                                       dropout=self.dropout if self.training else 0.0)
