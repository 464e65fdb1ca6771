"""Operator-level timing: one training step of the loss (forward + backward) through
warprnnt_pytorch.RNNTLoss, vs the reference operator's sequence of passes emulated on the same
library (full call into zeros-initialised grads, grads/=N, then grads.mul_(grad_output))."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "warp-transducer_b200"))
import warprnnt_pytorch.warp_rnnt as wr  # noqa: E402
from warprnnt_pytorch import RNNTLoss  # noqa: E402

N, T, L, V = 128, 150, 20, 5000
dev = torch.device("cuda:0")
acts = torch.rand((N, T, L + 1, V), device=dev, requires_grad=True)
labels = torch.as_tensor(np.random.default_rng(1).integers(1, V, size=(N, L)).astype(np.int32)).to(dev)
tl = torch.full((N,), T, dtype=torch.int32, device=dev)
ul = torch.full((N,), L, dtype=torch.int32, device=dev)
loss_fn = RNNTLoss(reduction='mean')


def ours():
    acts.grad = None
    loss = loss_fn(acts, labels, tl, ul)
    loss.backward()


def reference_style():
    a = acts.detach()
    grads = torch.zeros_like(a)                       # __init__.py:24
    costs = torch.empty(N, device=dev)
    wr.gpu_rnnt_async(a, labels, tl, ul, costs, grads, 0)
    costs = costs.sum().unsqueeze_(-1)
    costs /= N
    grads /= N                                        # :38-40
    grads.mul_(torch.ones(1, device=dev).view(-1, 1, 1, 1))   # backward :47-50


for name, fn in (("warprnnt_pytorch step", ours), ("reference operator's pass structure", reference_style)):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    print("%-40s %.3f ms/step  %.0f utt/s" % (name, ms, N / ms * 1e3))
