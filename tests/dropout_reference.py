"""Reference of the fused joiner's dropout on h (DESIGN.md §16, include/rnnt.h struct rnntJoinerDropout), for the
tests: a vectorised numpy Philox4x32-10 and the keep mask it defines, h~ from torch's own bf16 h, and the fp64
factors and gradients of the joiner with h~ as the logits' operand.

    key  = (lo32(seed), hi32(seed))
    ctr  = (k >> 2, c, 0, 0), c = (b U + u) T + t, the cell's dense index in the padded [N, U, T] grid
    keep = word (k & 3) of Philox4x32-10(ctr, key) >= floor(p 2^32), p as the float32 the C-ABI takes
    h~   = keep ? round_bf16(fp32(h) scale) : 0, scale = float32(1 / (1 - p))
    ds   = (dlogits W) act'(h) keep scale, act' from the undropped rounded h

Test infrastructure only.
"""
import numpy as np
import torch

import joiner_reference as jr
import pruned_joiner_reference as pjr

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)
_32 = np.uint64(32)


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11; Random123's philox4x32 with 10 rounds) on broadcastable arrays: ctr is
    four arrays of 32-bit words, key two.  Returns the four output words as uint64 arrays below 2^32."""
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint64) & _LO for x in ctr)
    k0, k1 = (np.asarray(x, dtype=np.uint64) & _LO for x in key)
    for i in range(10):
        if i:
            k0, k1 = (k0 + _W0) & _LO, (k1 + _W1) & _LO
        p0, p1 = _M0 * c0, _M1 * c2          # exact: both factors are below 2^32
        c0, c1, c2, c3 = (p1 >> _32) ^ c1 ^ k0, p1 & _LO, (p0 >> _32) ^ c3 ^ k1, p0 & _LO
    return c0, c1, c2, c3


def threshold(p):
    """floor(p 2^32) of the float32 p."""
    return int(np.floor(float(np.float32(p)) * 2.0 ** 32))


def scale(p):
    """float32(1 / (1 - p)) of the float32 p, as a Python float."""
    return float(np.float32(1.0 / (1.0 - float(np.float32(p)))))


def seed_key(seed):
    s = int(seed) & (2 ** 64 - 1)    # an int64 seed's two's-complement bits
    return s & 0xFFFFFFFF, s >> 32


def keep_mask(seed, N, T, U, H, p):
    """bool [N, T, U, H]: True where element k of cell (b, t, u) is kept."""
    b, t, u = np.meshgrid(np.arange(N), np.arange(T), np.arange(U), indexing="ij")
    c = ((b * U + u) * T + t).astype(np.uint64)[..., None]          # [N, T, U, 1]
    q = np.arange(H // 4, dtype=np.uint64)                         # [H / 4]
    words = philox4x32_10((q, c, 0, 0), seed_key(seed))
    x = np.stack(np.broadcast_arrays(*words), axis=-1).reshape(N, T, U, H)   # word k & 3 of counter k >> 2
    return torch.from_numpy(x >= np.uint64(threshold(p)))


def dropped_hidden(h, mask, p):
    """h~ [N, T, U, H] bf16 from the bf16 h and the keep mask (on h's device)."""
    kept = (h.float() * scale(p)).to(torch.bfloat16)
    return torch.where(mask.to(h.device), kept, torch.zeros_like(kept))


def act_grad(h, mask, p, activation):
    """fp64 act'(s) keep scale, act' from the undropped rounded h as the kernels take it."""
    return jr.act_grad(h, activation) * mask.to(h.device).double() * scale(p)


def log_probs(ht, weight, bias, labels, act_lens, label_lens, blank=0):
    """fp64 (px, py) of the joiner with h~ as the logits' operand."""
    return jr.log_probs(ht, weight, bias, labels, act_lens, label_lens, blank)


def gradients(h, ht, mask, p, weight, bias, labels, act_lens, label_lens, dpx, dpy, activation, blank=0):
    """fp64 (d_enc, d_pred, d_weight, d_bias): dW and dbias from h~, ds through act' keep scale."""
    dl = jr.dlogits(ht, weight, bias, labels, act_lens, label_lens, dpx, dpy, blank)
    ds = (dl @ weight.double()) * act_grad(h, mask, p, activation)
    return ds.sum(2), ds.sum(1), torch.einsum('ntuv,ntuh->vh', dl, ht.double()), dl.sum((0, 1, 2))


def pruned_log_probs(ht, weight, bias, labels, act_lens, label_lens, ranges, s_range, blank=0):
    """fp64 (px, py) of the pruned lattice: the dense ones on the covered cells, -inf elsewhere."""
    return pjr.log_probs(ht, weight, bias, labels, act_lens, label_lens, ranges, s_range, blank)


def pruned_gradients(h, ht, mask, p, weight, bias, labels, act_lens, label_lens, dpx, dpy, ranges, s_range,
                     activation, blank=0):
    """The dense gradients of the incoming gradients masked to the covered cells."""
    gx, gy = pjr.masked_incoming(dpx, dpy, ranges, s_range, act_lens, label_lens)
    return gradients(h, ht, mask, p, weight, bias, labels, act_lens, label_lens, gx, gy, activation, blank)
