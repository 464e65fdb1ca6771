"""Training-step time and peak memory of the pruned fused joiner (DESIGN.md §15) against the eager pruned recipe and
the fused dense joiner (dev tool, not the bench).  Per workload, in one process, interleaved round by round in a
rotating order:
  fused_pruned  pruned_joiner_rnnt_loss(enc, pred, weight, bias, ..., ranges, R) forward + backward through autograd
  eager_pruned  prune_joint_inputs(enc, pred, ranges, R), torch's bf16 joiner on them,
                logits = F.linear(tanh(enc_p + pred_p), weight, bias) [N, T, R, V], then this library's bf16
                pruned_rnnt_loss, forward + backward through autograd
  fused_dense   joiner_rnnt_loss(enc, pred, weight, bias, ...) over the whole [T, U] lattice
All start from bf16 enc, pred, weight and bias leaves and end with their four gradients.  The ranges (R = 5) come
once, before timing, from add_joint_rnnt_loss_with_ranges on random additive-joint projections, as in
tools/pruned_time.py; the simple loss itself is not timed.

    python tools/pruned_joiner_time.py [--rounds 3] [--steps 3] [--profile] [p1 p2 p3 p4]

Prints one JSON line: the GPU, its power limit, and per workload and arm the median ms per step over the rounds and
torch.cuda.max_memory_allocated over one step.  --profile adds, from a separate torch.profiler run, each kernel's
device ms per step in the fused pruned arm, with the GEMMs' achieved TFLOP/s (2 N T R H V FLOPs per GEMM).
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
from joiner_time import GEMMS, PEAK_TFLOPS, peak_bytes  # noqa: E402

R = 5
# name -> (N, T, U, H, V)
WORKLOADS = {
    "p1": (32, 250, 61, 512, 500),
    "p2": (128, 150, 21, 640, 5000),
    "p3": (64, 500, 101, 640, 5000),
    "p4": (64, 500, 101, 640, 32000),
}


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
    with torch.no_grad():
        am = torch.randn((N, T, V), device=dev, generator=gen)
        lm = torch.randn((N, U, V), device=dev, generator=gen)
        _, ranges = w.add_joint_rnnt_loss_with_ranges(am, lm, labels, tl, ul, R)
    del am, lm
    torch.cuda.empty_cache()
    return enc, pred, weight, bias, labels, tl, ul, ranges


def arms(name, dev):
    enc, pred, weight, bias, labels, tl, ul, ranges = inputs(name, dev)
    leaves = (enc, pred, weight, bias)

    def fused_pruned():
        for x in leaves:
            x.grad = None
        w.pruned_joiner_rnnt_loss(enc, pred, weight, bias, labels, tl, ul, ranges, R).backward()

    def eager_pruned():
        for x in leaves:
            x.grad = None
        enc_p, pred_p = w.prune_joint_inputs(enc, pred, ranges, R)
        logits = F.linear(torch.tanh(enc_p + pred_p), weight, bias)
        w.pruned_rnnt_loss(logits, labels, tl, ul, ranges).backward()

    def fused_dense():
        for x in leaves:
            x.grad = None
        w.joiner_rnnt_loss(enc, pred, weight, bias, labels, tl, ul).backward()

    return {"fused_pruned": fused_pruned, "eager_pruned": eager_pruned, "fused_dense": fused_dense}


def kernel_profile(fn, name, steps):
    from torch.profiler import ProfilerActivity, profile
    N, T, U, H, V = WORKLOADS[name]
    flops = 2.0 * N * T * R * H * V
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_time_total <= 0:
            continue
        k = next((g for g in GEMMS if g in e.key), None) or e.key[:60]
        ms = e.device_time_total / 1000.0 / steps
        out[k] = {"ms_per_step": round(out.get(k, {}).get("ms_per_step", 0.0) + ms, 3)}
        if k in GEMMS:
            tf = flops / (out[k]["ms_per_step"] * 1e-3) / 1e12
            out[k].update(tflops=round(tf, 1), share_of_989=round(tf / PEAK_TFLOPS, 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("workloads", nargs="*", default=list(WORKLOADS))
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0), "rounds": args.rounds,
           "steps_per_round": args.steps, "s_range": R}
    for name in args.workloads:
        N, T, U, H, V = WORKLOADS[name]
        fns = arms(name, dev)
        res = {"shape": dict(N=N, T=T, U=U, H=H, V=V, R=R),
               "eager_pruned_logits_and_grad_gb_from_shapes": round(2 * N * T * R * V * 2 / 1e9, 2)}
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
        res["fused_pruned_over_eager_pruned"] = round(res["ms_per_step"]["fused_pruned"] /
                                                      res["ms_per_step"]["eager_pruned"], 3)
        if args.profile:
            res["fused_pruned_kernels"] = kernel_profile(fns["fused_pruned"], name, 2)
        out[name] = res
        del fns
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
