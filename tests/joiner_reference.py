"""fp64 torch reference of the fused joiner (DESIGN.md §14, include/rnnt.h rnnt_b200_joiner_forward / _backward), for
the tests.  Runs on whatever device its tensors are on.

    h = round_bf16(act(fp32(enc[b,t]) + fp32(pred[b,u])))      (hidden: formed by torch, passed in by the caller)
    logits = h W^T + bias in fp64, lp = log_softmax(logits)
    py[b,u,t] = lp[b,t,u,blank], px[b,u,t] = lp[b,t,u,labels[b,u]]   (-inf on padding, NaN for a label outside [0, V))

and the gradients of the four inputs from incoming dpx, dpy, with act' taken from the rounded h (tanh: 1 - h^2,
relu: [h > 0]) as the kernels take it.  Padding: t >= T_b = clip(act_lens, 1, T); u > S_b for py, u >= S_b for px,
S_b = clip(label_lens, 0, U-1).  Test infrastructure only.
"""
import torch


def hidden(enc, pred, activation):
    """[N, T, U, H] bf16 h, formed in fp32 and rounded once to nearest."""
    s = enc.float()[:, :, None, :] + pred.float()[:, None, :, :]
    a = torch.tanh(s) if activation == 'tanh' else torch.relu(s)
    return a.to(torch.bfloat16)


def masks(act_lens, label_lens, T, U):
    """(cell [N, T, U], label [N, T, U-1]) validity masks."""
    dev = act_lens.device
    tb = act_lens.long().clamp(1, T)
    sb = label_lens.long().clamp(0, U - 1)
    t = torch.arange(T, device=dev)[None, :, None]
    u = torch.arange(U, device=dev)[None, None, :]
    cell = (t < tb[:, None, None]) & (u <= sb[:, None, None])
    lab = (t < tb[:, None, None]) & (u[..., :U - 1] < sb[:, None, None])
    return cell, lab


def logits(h, weight, bias):
    """fp64 [N, T, U, V] logits of a bf16 h."""
    z = h.double() @ weight.double().T
    return z + bias.double() if bias is not None else z


def log_probs(h, weight, bias, labels, act_lens, label_lens, blank=0):
    """fp64 (px [N, U-1, T], py [N, U, T])."""
    N, T, U, _ = h.shape
    V = weight.shape[0]
    lp = torch.log_softmax(logits(h, weight, bias), -1)
    cell, lab = masks(act_lens, label_lens, T, U)
    py = lp[..., blank].masked_fill(~cell, -float('inf'))
    lbl = labels.long()
    inside = (lbl >= 0) & (lbl < V)
    g = lp[:, :, :U - 1, :].gather(-1, lbl.clamp(0, V - 1)[:, None, :, None].expand(N, T, U - 1, 1))[..., 0]
    g = torch.where(inside[:, None, :], g, torch.full_like(g, float('nan')))
    px = g.masked_fill(~lab, -float('inf'))
    return px.permute(0, 2, 1).contiguous(), py.permute(0, 2, 1).contiguous()


def dlogits(h, weight, bias, labels, act_lens, label_lens, dpx, dpy, blank=0):
    """fp64 [N, T, U, V] d/dlogits of sum(dpx px) + sum(dpy py), zero on padding cells."""
    N, T, U, _ = h.shape
    V = weight.shape[0]
    p = torch.softmax(logits(h, weight, bias), -1)
    cell, lab = masks(act_lens, label_lens, T, U)
    gy = dpy.double().permute(0, 2, 1) * cell                       # [N, T, U]
    gx = torch.zeros_like(gy)
    gx[..., :U - 1] = dpx.double().permute(0, 2, 1) * lab
    d = -(gx + gy)[..., None] * p
    d[..., blank] += gy
    lbl = labels.long()
    inside = ((lbl >= 0) & (lbl < V))[:, None, :, None]
    onehot = torch.zeros(N, T, U - 1, V, dtype=torch.float64, device=h.device)
    onehot.scatter_(-1, lbl.clamp(0, V - 1)[:, None, :, None].expand(N, T, U - 1, 1), 1.0)
    d[..., :U - 1, :] += gx[..., :U - 1, None] * onehot * inside
    return d


def act_grad(h, activation):
    hd = h.double()
    return 1.0 - hd * hd if activation == 'tanh' else (hd > 0).double()


def gradients(h, weight, bias, labels, act_lens, label_lens, dpx, dpy, activation, blank=0, dl=None):
    """fp64 (d_enc [N, T, H], d_pred [N, U, H], d_weight [V, H], d_bias [V]) from the factors' gradients."""
    if dl is None:
        dl = dlogits(h, weight, bias, labels, act_lens, label_lens, dpx, dpy, blank)
    hd = h.double()
    dw = torch.einsum('ntuv,ntuh->vh', dl, hd)
    db = dl.sum((0, 1, 2))
    ds = (dl @ weight.double()) * act_grad(h, activation)
    return ds.sum(2), ds.sum(1), dw, db


def fp64_forward(enc, pred, weight, bias, labels, act_lens, label_lens, activation, blank=0):
    """The same function entirely in fp64 without rounding h, differentiable by autograd: what the explicit
    gradients above are when h is not rounded."""
    s = enc[:, :, None, :] + pred[:, None, :, :]
    h = torch.tanh(s) if activation == 'tanh' else torch.relu(s)
    z = h @ weight.T + (bias if bias is not None else 0)
    N, T, U, V = z.shape
    lp = torch.log_softmax(z, -1)
    cell, lab = masks(act_lens, label_lens, T, U)
    py = torch.where(cell, lp[..., blank], torch.full_like(lp[..., blank], -float('inf')))
    g = lp[:, :, :U - 1, :].gather(-1, labels.long()[:, None, :, None].expand(N, T, U - 1, 1))[..., 0]
    px = torch.where(lab, g, torch.full_like(g, -float('inf')))
    return px.permute(0, 2, 1), py.permute(0, 2, 1)
