"""Device time of one training step of the dense RNN-T loss, of the pruned loss (DESIGN.md §8) at R = 4 and 8, and
of the simple (additive-joint) loss plus its pruning ranges, interleaved round by round in a rotating order (dev
tool, not the bench).

    python tools/pruned_time.py [--rounds 5] [--steps 10] [c3 long ...]

Prints one JSON line: the GPU, its power limit, and per workload and logits dtype (fp32, bf16) the median ms per
step of each setting, and the streaming passes' (pass 1 + pass 2) achieved GB/s on 3 x element size per logit
(12 B for fp32) from the per-kernel events of the profiling mode.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "warp-transducer_b200"))
import warprnnt_pytorch.warp_rnnt as wr  # noqa: E402
from warprnnt_pytorch import joint, pruned  # noqa: E402

CFG = {"c3": (128, 150, 20, 5000), "long": (32, 500, 150, 500)}   # N, T, max label length, V
CODE = {torch.float32: 0, torch.bfloat16: 1}


def power_limit_w(index):
    try:
        import pynvml
        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetPowerManagementLimit(pynvml.nvmlDeviceGetHandleByIndex(index)) / 1000.0
    except Exception:
        return None


def step_ms(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def pass_ms(fn, steps):
    """mean (rowstats + grad) ms over `steps` profiled calls: the two streaming passes of the call"""
    wr.set_profiling(True)
    wr.profile_collect()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    _, (ms1, _, ms2) = wr.profile_collect()
    wr.set_profiling(False)
    return ms1 + ms2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("workloads", nargs="*", default=["c3", "long"])
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = wr.lib()
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
        ranges = torch.empty((N, T), dtype=torch.int32, device=dev)
        opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream(dev).cuda_stream, blank_label=0,
                             maxT=T, maxU=U, batch_first=True)

        def simple():
            ws = joint.add_joint_call(trans, pred, labels, tl, ul, costs, dtrans, dpred, 0, 1.0)
            lib.rnnt_b200_add_joint_prune_ranges(ul.data_ptr(), tl.data_ptr(), N, 4, ranges.data_ptr(),
                                                 ws.data_ptr(), opt)

        simple()
        torch.cuda.synchronize()
        ranges4 = ranges.clone()
        for tag, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
            esz = torch.tensor([], dtype=dt).element_size()
            acts = torch.rand((N, T, U, V), device=dev, generator=gen).to(dt)
            grads = torch.empty_like(acts)
            ws_d = torch.empty(wr.workspace_size(T, U, N, 4), dtype=torch.uint8, device=dev)
            fns = {"dense": lambda: wr.gpu_rnnt_async(acts, labels, tl, ul, costs, grads, 0, 1.0, ws_d),
                   "simple_and_ranges": simple}
            logit_count = {"dense": N * T * U * V}
            bufs = []
            for R in (4, 8):
                x = torch.rand((N, T, R, V), device=dev, generator=gen).to(dt)
                g = torch.empty_like(x)
                rg = ranges4 if R == 4 else torch.clamp(ranges4 - 2, min=0).contiguous()
                ws = torch.empty(pruned.pruned_workspace_size(T, U, R, N, 4), dtype=torch.uint8, device=dev)
                bufs.append((x, g, rg, ws))

                def fn(x=x, g=g, rg=rg, ws=ws, R=R):
                    st = lib.rnnt_b200_pruned_loss_async_ex(CODE[dt], 0, x.data_ptr(), g.data_ptr(), rg.data_ptr(), R,
                                                            labels.data_ptr(), ul.data_ptr(), tl.data_ptr(), V, N,
                                                            costs.data_ptr(), 1.0, wr.rnntGradOptions(), ws.data_ptr(),
                                                            opt)
                    assert st == 0, wr.status_string(st)
                fns["pruned_R%d" % R] = fn
                logit_count["pruned_R%d" % R] = N * T * R * V
            names = list(fns)
            ms = {k: [] for k in names}
            for r in range(args.rounds):
                for k in names[r % len(names):] + names[:r % len(names)]:
                    ms[k].append(step_ms(fns[k], args.steps))
            med = {k: float(np.median(v)) for k, v in ms.items()}
            gbs = {k: logit_count[k] * 3 * esz / (pass_ms(fns[k], args.steps) * 1e-3) / 1e9 for k in logit_count}
            out["%s_%s" % (name, tag)] = {"ms_per_step": med, "all_ms": ms, "passes_GBps": gbs,
                                          "logits_GB": {k: n * esz / 1e9 for k, n in logit_count.items()}}
            del acts, grads, bufs, fns
            torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
