"""Device time of one loss+grad step (async C-ABI) without gradient options, with FastEmit only and with FastEmit
plus clamp, the three settings interleaved round by round in a rotating order (dev tool, not the bench).

    python tools/grad_options_time.py [--lambda 0.01] [--clamp 0.001] [--rounds 5] [--steps 10] [c3 ...]

Prints one JSON line: the GPU, its power limit, and per workload and logits dtype (fp32, bf16) the median ms per
step of each setting over the rounds and its change against the step without options.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "warp-transducer_b200"))
import warprnnt_pytorch.warp_rnnt as wr  # noqa: E402

CFG = {"c2": (128, 150, 40, 28), "c3": (128, 150, 20, 5000), "c4": (64, 1500, 300, 50)}


def power_limit_w(index):
    try:
        import pynvml
        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(index)) / 1000.0
    except Exception:
        return None


def step_ms(fn, steps, flush):
    """ms per step on the current stream (CUDA events); with `flush` the L2 is overwritten before every step."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    if flush is None:
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps
    total = 0.0
    for _ in range(steps):
        flush.zero_()
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        total += e0.elapsed_time(e1)
    return total / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lambda", dest="lam", type=float, default=0.01)
    ap.add_argument("--clamp", type=float, default=0.001)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("workloads", nargs="*", default=["c3"])
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    settings = {"off": (0.0, -1.0), "fastemit": (args.lam, -1.0), "fastemit_clamp": (args.lam, args.clamp)}
    names = list(settings)
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0), "rounds": args.rounds,
           "steps_per_round": args.steps, "fastemit_lambda": args.lam, "clamp": args.clamp}
    for name in args.workloads:
        N, T, L, V = CFG[name]
        U = L + 1
        rng = np.random.default_rng(1)
        labels = torch.as_tensor(rng.integers(1, V, size=(N, L)).astype(np.int32)).to(dev)
        tl = torch.full((N,), T, dtype=torch.int32, device=dev)
        ul = torch.full((N,), L, dtype=torch.int32, device=dev)
        costs = torch.empty(N, device=dev)
        ws = torch.empty(wr.workspace_size(T, U, N, 4), dtype=torch.uint8, device=dev)
        for tag, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
            acts = torch.rand((N, T, U, V), device=dev, generator=torch.Generator(dev).manual_seed(7)).to(dt)
            grads = torch.empty_like(acts)
            flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev) \
                if acts.numel() * acts.element_size() < (1 << 30) else None
            ms = {k: [] for k in names}
            for r in range(args.rounds):
                for k in names[r % len(names):] + names[:r % len(names)]:
                    lam, c = settings[k]
                    ms[k].append(step_ms(lambda: wr.gpu_rnnt_async(acts, labels, tl, ul, costs, grads, 0, 1.0, ws,
                                                                   fastemit_lambda=lam, clamp=c), args.steps, flush))
            med = {k: float(np.median(v)) for k, v in ms.items()}
            out["%s_%s" % (name, tag)] = {"ms_per_step": med, "all_ms": ms,
                                          "vs_off": {k: med[k] / med["off"] - 1.0 for k in names if k != "off"}}
            del acts, grads, flush
            torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
