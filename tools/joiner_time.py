"""Training-step time and peak memory of the fused joiner (DESIGN.md §14) against the eager joiner (dev tool, not the
bench).  Per workload, in one process, interleaved round by round in a rotating order:
  fused   joiner_rnnt_loss(enc, pred, weight, bias, ...) forward + backward through autograd
  eager   torch's bf16 joiner, logits = F.linear(tanh(enc[:, :, None] + pred[:, None]), weight, bias) [N, T, U, V],
          then this library's bf16 rnnt_loss on them, forward + backward through autograd
Both start from bf16 enc, pred, weight and bias leaves and end with their four gradients.

    python tools/joiner_time.py [--rounds 5] [--steps 5] [--profile] [j1 j2 j3]

Prints one JSON line: the GPU, its power limit, and per workload and arm the median ms per step over the rounds and
torch.cuda.max_memory_allocated over one step.  J3 runs the fused arm only; its eager footprint is stated from shapes
(bf16 logits and their gradient).  --profile adds, from a separate torch.profiler run, each joiner kernel's device
ms per step and its achieved TFLOP/s from FLOPs computed from shapes (2 cells H V per GEMM), against the H100 SXM's
989 TFLOP/s dense bf16 data-sheet figure.
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

# name -> (N, T, U, H, V)
WORKLOADS = {
    "j1": (32, 250, 61, 512, 500),
    "j2": (128, 150, 21, 640, 5000),
    "j3": (64, 500, 101, 640, 5000),
}
FUSED_ONLY = {"j3"}
GEMMS = ("joiner_lse_kernel", "joiner_dlogits_kernel", "joiner_ds_kernel", "joiner_dw_kernel")
PEAK_TFLOPS = 989.0


def inputs(name, dev):
    N, T, U, H, V = WORKLOADS[name]
    gen = torch.Generator(dev).manual_seed(3)
    enc = torch.randn((N, T, H), device=dev, generator=gen).to(torch.bfloat16).requires_grad_(True)
    pred = torch.randn((N, U, H), device=dev, generator=gen).to(torch.bfloat16).requires_grad_(True)
    weight = (torch.randn((V, H), device=dev, generator=gen) / H ** 0.5).to(torch.bfloat16).requires_grad_(True)
    bias = torch.zeros(V, device=dev).to(torch.bfloat16).requires_grad_(True)
    labels = torch.randint(1, V, (N, U - 1), device=dev, generator=gen, dtype=torch.int32)
    tl = torch.full((N,), T, dtype=torch.int32, device=dev)
    ul = torch.full((N,), U - 1, dtype=torch.int32, device=dev)
    return enc, pred, weight, bias, labels, tl, ul


def arms(name, dev):
    enc, pred, weight, bias, labels, tl, ul = inputs(name, dev)
    leaves = (enc, pred, weight, bias)

    def fused():
        for x in leaves:
            x.grad = None
        w.joiner_rnnt_loss(enc, pred, weight, bias, labels, tl, ul).backward()

    def eager():
        for x in leaves:
            x.grad = None
        logits = F.linear(torch.tanh(enc[:, :, None, :] + pred[:, None, :, :]), weight, bias)
        w.rnnt_loss(logits, labels, tl, ul).backward()

    return {"fused": fused} if name in FUSED_ONLY else {"fused": fused, "eager": eager}


def peak_bytes(fn, dev):
    fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated(dev), base


def gemm_profile(fn, name, steps):
    from torch.profiler import ProfilerActivity, profile
    N, T, U, H, V = WORKLOADS[name]
    flops = 2.0 * N * T * U * H * V
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        k = next((g for g in GEMMS if g in e.key), None)
        if k is None and "joiner_" not in e.key:
            continue
        ms = e.device_time_total / 1000.0 / steps
        k = k or e.key[:60]
        out[k] = {"ms_per_step": round(ms, 3)}
        if k in GEMMS and ms > 0:
            tf = flops / (ms * 1e-3) / 1e12
            out[k].update(tflops=round(tf, 1), share_of_989=round(tf / PEAK_TFLOPS, 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("workloads", nargs="*", default=list(WORKLOADS))
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0), "rounds": args.rounds,
           "steps_per_round": args.steps}
    for name in args.workloads:
        N, T, U, H, V = WORKLOADS[name]
        fns = arms(name, dev)
        res = {"shape": dict(N=N, T=T, U=U, H=H, V=V)}
        for k, fn in fns.items():
            peak, base = peak_bytes(fn, dev)
            res.setdefault("peak_gb", {})[k] = round(peak / 1e9, 3)
            res.setdefault("resident_before_step_gb", {})[k] = round(base / 1e9, 3)
        ms = {k: [] for k in fns}
        names = list(fns)
        for r in range(args.rounds):
            for k in names[r % len(names):] + names[:r % len(names)]:
                ms[k].append(step_ms(fns[k], args.steps))
        res["ms_per_step"] = {k: round(float(np.median(v)), 3) for k, v in ms.items()}
        res["all_ms"] = {k: [round(x, 3) for x in v] for k, v in ms.items()}
        if "eager" in res["ms_per_step"]:
            res["fused_over_eager"] = round(res["ms_per_step"]["fused"] / res["ms_per_step"]["eager"], 3)
        else:
            res["eager_logits_and_grad_gb_from_shapes"] = round(2 * N * T * U * V * 2 / 1e9, 1)
        if args.profile:
            res["fused_kernels"] = gemm_profile(fns["fused"], name, 2)
        out[name] = res
        del fns
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
