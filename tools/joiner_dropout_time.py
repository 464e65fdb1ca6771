"""Training-step time and peak memory of the fused joiners with dropout on the hidden activation (DESIGN.md §16)
against the same calls without it, and against NeMo's eager joint with dropout (dev tool, not the bench).  Per
workload, in one process, interleaved round by round in a rotating order:
  fused_p0      joiner_rnnt_loss(..., activation) forward + backward (pruned_joiner_rnnt_loss on P2)
  fused_p02     the same with dropout=0.2 (a fresh seed per step, drawn on the device)
  eager_p02     NeMo's joint: logits = F.linear(F.dropout(act(enc[:, :, None] + pred[:, None]), 0.2), weight, bias)
                [N, T, U, V], then this library's bf16 rnnt_loss on them (dense workloads only)
All start from bf16 enc, pred, weight and bias leaves and end with their four gradients.  P2's ranges (R = 5) come
once, before timing, from add_joint_rnnt_loss_with_ranges, as in tools/pruned_joiner_time.py.  act is relu (NeMo's
default) or, with --activation tanh, tanh, whose ds epilogue recomputes h under dropout.

    python tools/joiner_dropout_time.py [--rounds 5] [--steps 5] [--activation relu] [--no-eager] [--profile]
                                        [j1 j2 p2]

Prints one JSON line: the GPU, its power limit, and per workload and arm the median ms per step over the rounds and
torch.cuda.max_memory_allocated over one step, with fused_p02 / fused_p0.  --profile adds, from a separate
torch.profiler run, each joiner kernel's device ms per step in the two fused arms.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "warp-transducer_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import warprnnt_pytorch as w  # noqa: E402
from delay_time import power_limit_w, step_ms  # noqa: E402
from joiner_time import peak_bytes  # noqa: E402

P, R = 0.2, 5
# name -> (N, T, U, H, V, pruned)
WORKLOADS = {
    "j1": (32, 250, 61, 512, 500, False),
    "j2": (128, 150, 21, 640, 5000, False),
    "p2": (128, 150, 21, 640, 5000, True),
}


def inputs(name, dev):
    N, T, U, H, V, pruned = WORKLOADS[name]
    gen = torch.Generator(dev).manual_seed(3)
    enc = torch.randn((N, T, H), device=dev, generator=gen).to(torch.bfloat16).requires_grad_(True)
    pred = torch.randn((N, U, H), device=dev, generator=gen).to(torch.bfloat16).requires_grad_(True)
    weight = (torch.randn((V, H), device=dev, generator=gen) / H ** 0.5).to(torch.bfloat16).requires_grad_(True)
    bias = torch.zeros(V, device=dev).to(torch.bfloat16).requires_grad_(True)
    labels = torch.randint(1, V, (N, U - 1), device=dev, generator=gen, dtype=torch.int32)
    tl = torch.full((N,), T, dtype=torch.int32, device=dev)
    ul = torch.full((N,), U - 1, dtype=torch.int32, device=dev)
    ranges = None
    if pruned:
        with torch.no_grad():
            am = torch.randn((N, T, V), device=dev, generator=gen)
            lm = torch.randn((N, U, V), device=dev, generator=gen)
            _, ranges = w.add_joint_rnnt_loss_with_ranges(am, lm, labels, tl, ul, R)
        del am, lm
        torch.cuda.empty_cache()
    return enc, pred, weight, bias, labels, tl, ul, ranges


def arms(name, dev, eager, activation):
    enc, pred, weight, bias, labels, tl, ul, ranges = inputs(name, dev)
    leaves = (enc, pred, weight, bias)

    def fused(p):
        def step():
            for x in leaves:
                x.grad = None
            if ranges is None:
                loss = w.joiner_rnnt_loss(enc, pred, weight, bias, labels, tl, ul, activation=activation, dropout=p)
            else:
                loss = w.pruned_joiner_rnnt_loss(enc, pred, weight, bias, labels, tl, ul, ranges, R,
                                                 activation=activation, dropout=p)
            loss.backward()
        return step

    def eager_p02():
        for x in leaves:
            x.grad = None
        s = enc[:, :, None, :] + pred[:, None, :, :]
        h = F.dropout(torch.relu(s) if activation == "relu" else torch.tanh(s), P)
        w.rnnt_loss(F.linear(h, weight, bias), labels, tl, ul).backward()

    fns = {"fused_p0": fused(0.0), "fused_p02": fused(P)}
    if eager and ranges is None:
        fns["eager_p02"] = eager_p02
    return fns


def kernel_ms(fn, steps):
    """Device ms per step of each joiner kernel (torch.profiler, CUDA activity only)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    return {e.key[:70]: round(e.device_time_total / 1000.0 / steps, 3) for e in prof.key_averages()
            if "joiner_" in e.key}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--activation", default="relu", choices=["relu", "tanh"])
    ap.add_argument("--no-eager", action="store_true")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("workloads", nargs="*", default=list(WORKLOADS))
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0), "rounds": args.rounds,
           "steps_per_round": args.steps, "dropout": P, "activation": args.activation}
    for name in args.workloads:
        N, T, U, H, V, pruned = WORKLOADS[name]
        fns = arms(name, dev, not args.no_eager, args.activation)
        res = {"shape": dict(N=N, T=T, U=U, H=H, V=V, **({"R": R} if pruned else {}))}
        for k, fn in fns.items():
            peak, _ = peak_bytes(fn, dev)
            res.setdefault("peak_gb", {})[k] = round(peak / 1e9, 3)
        ms = {k: [] for k in fns}
        names = list(fns)
        for r in range(args.rounds):
            for k in names[r % len(names):] + names[:r % len(names)]:
                ms[k].append(step_ms(fns[k], args.steps))
        res["ms_per_step"] = {k: round(float(np.median(v)), 3) for k, v in ms.items()}
        res["all_ms"] = {k: [round(x, 3) for x in v] for k, v in ms.items()}
        res["p02_over_p0"] = round(res["ms_per_step"]["fused_p02"] / res["ms_per_step"]["fused_p0"], 3)
        if args.profile:
            res["kernels_ms"] = {k: kernel_ms(fns[k], 2) for k in ("fused_p0", "fused_p02")}
        out[name] = res
        del fns
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
