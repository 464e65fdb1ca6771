"""Device time of forced alignment (DESIGN.md §12) against the alpha-only forward it shares pass 1 with (dev tool,
not the bench).  Per workload, in one process, the two calls interleaved round by round in a rotating order:
  align     rnnt_b200_align (or rnnt_b200_pruned_align): pass 1, the Viterbi wavefront and its backtrace
  forward   rnnt_b200_forward_topo with prepare_backward = 0 (or the pruned forward): pass 1 and the alpha wavefront

    python tools/align_time.py [--rounds 7] [--steps 10] [--profile] [c2_fp32 c3_fp32 c3_bf16 c4_fp32 c3_pruned5]

Prints one JSON line: the GPU, its power limit, and per workload the median ms per call of each over the rounds and
the change of "align" against "forward".  --profile adds, from a separate torch.profiler run of each workload, the
mean device time of every kernel the two calls launch.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "warp-transducer_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import warprnnt_pytorch.warp_rnnt as wr  # noqa: E402
from delay_time import power_limit_w, step_ms  # noqa: E402
from warprnnt_pytorch import pruned  # noqa: E402

# name -> (N, T, max label length, V, storage, s_range or None)
WORKLOADS = {
    "c2_fp32": (128, 150, 40, 28, torch.float32, None),
    "c3_fp32": (128, 150, 20, 5000, torch.float32, None),
    "c3_bf16": (128, 150, 20, 5000, torch.bfloat16, None),
    "c4_fp32": (64, 1500, 300, 50, torch.float32, None),
    "c3_pruned5": (128, 150, 20, 5000, torch.float32, 5),
}
DTYPE = {torch.float32: wr.RNNT_B200_FP32, torch.bfloat16: wr.RNNT_B200_BF16}


def calls(name, dev):
    """{"align": fn, "forward": fn} of one workload, on fresh inputs."""
    N, T, L, V, dt, R = WORKLOADS[name]
    U = L + 1
    rng = np.random.default_rng(1)
    gen = torch.Generator(dev).manual_seed(7)
    labels = torch.as_tensor(rng.integers(1, V, size=(N, L)).astype(np.int32)).to(dev)
    tl = torch.full((N,), T, dtype=torch.int32, device=dev)
    ul = torch.full((N,), L, dtype=torch.int32, device=dev)
    acts = torch.rand((N, T, R or U, V), device=dev, generator=gen).to(dt)
    costs = torch.empty(N, device=dev)
    scores = torch.empty(N, device=dev)
    frames = torch.empty((N, L), dtype=torch.int32, device=dev)
    opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream(dev).cuda_stream, blank_label=0,
                         maxT=T, maxU=U, batch_first=True)
    lib, code = wr.lib(), DTYPE[dt]
    if R is None:
        ws = torch.empty(wr.workspace_size(T, U, N, 4), dtype=torch.uint8, device=dev)

        def align():
            st = lib.rnnt_b200_align(code, 0, acts.data_ptr(), labels.data_ptr(), ul.data_ptr(), tl.data_ptr(), V, N,
                                     0, frames.data_ptr(), scores.data_ptr(), ws.data_ptr(), opt)
            assert st == 0, wr.status_string(st)

        def forward():
            st = lib.rnnt_b200_forward_topo(code, acts.data_ptr(), labels.data_ptr(), ul.data_ptr(), tl.data_ptr(), V,
                                            N, costs.data_ptr(), 0, wr.rnntLatticeOptions(), 0, ws.data_ptr(), opt)
            assert st == 0, wr.status_string(st)
    else:
        # windows of width R spread evenly over the labels: every utterance keeps a path
        t = torch.arange(T, device=dev)
        ranges = (t * (U - R) // max(T - 1, 1)).to(torch.int32).expand(N, T).contiguous()
        ws = torch.empty(pruned.pruned_workspace_size(T, U, R, N, 4), dtype=torch.uint8, device=dev)

        def align():
            st = lib.rnnt_b200_pruned_align(code, acts.data_ptr(), ranges.data_ptr(), R, labels.data_ptr(),
                                            ul.data_ptr(), tl.data_ptr(), V, N, 0, frames.data_ptr(),
                                            scores.data_ptr(), ws.data_ptr(), opt)
            assert st == 0, wr.status_string(st)

        def forward():
            st = lib.rnnt_b200_pruned_forward_topo(code, acts.data_ptr(), ranges.data_ptr(), R, labels.data_ptr(),
                                                   ul.data_ptr(), tl.data_ptr(), V, N, costs.data_ptr(), 0,
                                                   wr.rnntLatticeOptions(), 0, ws.data_ptr(), opt)
            assert st == 0, wr.status_string(st)
    return {"align": align, "forward": forward}, (scores, costs)


def compare(fns, rounds, steps):
    names = list(fns)
    ms = {k: [] for k in names}
    for r in range(rounds):
        for k in names[r % len(names):] + names[:r % len(names)]:
            ms[k].append(step_ms(fns[k], steps))
    med = {k: float(np.median(v)) for k, v in ms.items()}
    return {"ms_per_call": med, "all_ms": ms, "align_vs_forward": med["align"] / med["forward"] - 1.0}


def kernel_ms(fns, steps):
    """Mean device ms per call of each kernel, per call kind, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for k, fn in fns.items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                fn()
            torch.cuda.synchronize()
        out[k] = {e.key[:90]: round(e.device_time_total / 1000.0 / steps, 4)
                  for e in prof.key_averages() if e.device_time_total > 0}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("workloads", nargs="*", default=list(WORKLOADS))
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0), "rounds": args.rounds,
           "steps_per_round": args.steps}
    for name in args.workloads:
        fns, (scores, costs) = calls(name, dev)
        res = compare(fns, args.rounds, args.steps)
        torch.cuda.synchronize()
        # the best path is one of the paths the loss sums over: score <= -cost
        res["score_le_minus_cost"] = bool((scores <= -costs * (1 - 1e-6) + 1e-3).all())
        if args.profile:
            res["kernel_ms"] = kernel_ms(fns, args.steps)
        out[name] = res
        del fns
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
