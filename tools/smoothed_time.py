"""Device time of one training step of the additive joint, plain and smoothed (DESIGN.md §9), through the C-ABI,
interleaved round by round in a rotating order (dev tool, not the bench).

    python tools/smoothed_time.py [--rounds 5] [--steps 10] [--kernels] [c3 long ...]

Settings: the plain joint step (forward + backward); the smoothed step at (lm_only_scale, am_only_scale) = (0.25, 0)
and (0.25, 0.1); the smoothed simple loss plus its pruning ranges (R = 4) at (0.25, 0).  Prints one JSON line: the
GPU, its power limit, and per workload the median ms per step of each setting.  --kernels adds, per setting, the
device time of each kernel in microseconds per step (torch.profiler, after the timed rounds).
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
from warprnnt_pytorch import joint  # noqa: E402
from pruned_time import CFG, power_limit_w, step_ms  # noqa: E402


def kernel_us(fn, steps):
    """{kernel name without its parameter list: device microseconds per step}"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    tot = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            key = e.name.split("(")[0].replace("void ", "").replace("b200rnnt::", "")
            tot[key] = tot.get(key, 0.0) + e.device_time / steps
    return dict(sorted(((k, round(v, 1)) for k, v in tot.items()), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--kernels", action="store_true", help="per-kernel device time of each setting (torch.profiler)")
    ap.add_argument("workloads", nargs="*", default=["c3", "long"])
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = joint._lib
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0), "rounds": args.rounds,
           "steps_per_round": args.steps}
    for name in args.workloads:
        N, T, L, V = CFG[name]
        U = L + 1
        rng = np.random.default_rng(1)
        labels = torch.as_tensor(rng.integers(1, V, size=(N, L)).astype(np.int32)).to(dev)
        tl = torch.full((N,), T, dtype=torch.int32, device=dev)
        ul = torch.full((N,), L, dtype=torch.int32, device=dev)
        costs = torch.empty(N, device=dev)
        gen = torch.Generator(dev).manual_seed(7)
        trans = torch.randn((N, T, V), device=dev, generator=gen)
        pred = torch.randn((N, U, V), device=dev, generator=gen)
        dtrans, dpred = torch.empty_like(trans), torch.empty_like(pred)
        grad_costs = torch.ones(N, device=dev)
        ranges = torch.empty((N, T), dtype=torch.int32, device=dev)
        opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream(dev).cuda_stream, blank_label=0,
                             maxT=T, maxU=U, batch_first=True)
        n = joint.C.c_size_t(0)
        assert lib.rnnt_b200_add_joint_smoothed_workspace_size(T, U, N, V, joint.C.byref(n)) == 0
        ws = torch.empty(n.value, dtype=torch.uint8, device=dev)
        gopt = wr.rnntGradOptions()
        args_f = (trans.data_ptr(), pred.data_ptr(), labels.data_ptr(), ul.data_ptr(), tl.data_ptr(), V, N)
        args_b = (trans.data_ptr(), pred.data_ptr(), dtrans.data_ptr(), dpred.data_ptr(), labels.data_ptr(),
                  ul.data_ptr(), tl.data_ptr(), V, N, grad_costs.data_ptr(), 1.0)

        def step(lm, am, with_ranges=False, backward=True):
            sm = joint.rnntSmoothOptions(lm, am)

            def fn():
                st = lib.rnnt_b200_add_joint_smoothed_forward(*args_f, costs.data_ptr(), 1, sm, ws.data_ptr(), opt)
                assert st == 0, wr.status_string(st)
                if with_ranges:
                    st = lib.rnnt_b200_add_joint_prune_ranges(ul.data_ptr(), tl.data_ptr(), N, 4, ranges.data_ptr(),
                                                              ws.data_ptr(), opt)
                    assert st == 0, wr.status_string(st)
                if backward:
                    st = lib.rnnt_b200_add_joint_smoothed_backward(*args_b, gopt, sm, ws.data_ptr(), opt)
                    assert st == 0, wr.status_string(st)
            return fn

        fns = {"plain": step(0.0, 0.0), "smoothed_0.25_0": step(0.25, 0.0), "smoothed_0.25_0.1": step(0.25, 0.1),
               "simple_and_ranges_0.25_0": step(0.25, 0.0, with_ranges=True)}
        names = list(fns)
        ms = {k: [] for k in names}
        for r in range(args.rounds):
            for k in names[r % len(names):] + names[:r % len(names)]:
                ms[k].append(step_ms(fns[k], args.steps))
        med = {k: float(np.median(v)) for k, v in ms.items()}
        out[name] = {"shape_NTUV": [N, T, U, V], "ms_per_step": med, "all_ms": ms,
                     "vs_plain": {k: med[k] / med["plain"] for k in names}}
        if args.kernels:
            out[name]["kernel_us_per_step"] = {k: kernel_us(fns[k], args.steps) for k in names}
        del ws, trans, pred, dtrans, dpred
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
