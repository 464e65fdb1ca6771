"""Device time of one training step with the regular and the modified topology (DESIGN.md §11), the two settings
interleaved round by round in a rotating order (dev tool, not the bench):
  dense    the full loss+grad call (async C-ABI) on fp32 and bf16 logits
  pruned   the full pruned call at R = 4 (fp32), windows from the simple loss of the same topology
  joint    the additive joint with its pruning ranges (forward, ranges, backward), plain and smoothed at (0.25, 0)

    python tools/modified_time.py [--rounds 7] [--steps 10] [c3 ...]

Prints one JSON line: the GPU, its power limit, and per workload and setting the median ms per step of each of
"regular" / "modified" over the rounds and the change of "modified" against "regular".  Every utterance has
T_b >= U_b - 1, so every modified lattice has a path.
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
from delay_time import CFG, power_limit_w, step_ms  # noqa: E402
from warprnnt_pytorch import pruned  # noqa: E402

TOPOS = {"regular": 0, "modified": 1}


def compare(fns, rounds, steps):
    names = list(fns)
    ms = {k: [] for k in names}
    for r in range(rounds):
        for k in names[r % len(names):] + names[:r % len(names)]:
            ms[k].append(step_ms(fns[k], steps))
    med = {k: float(np.median(v)) for k, v in ms.items()}
    return {"ms_per_step": med, "all_ms": ms, "modified_vs_regular": med["modified"] / med["regular"] - 1.0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("workloads", nargs="*", default=["c3"])
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = wr.lib()
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(0), "rounds": args.rounds,
           "steps_per_round": args.steps}
    for name in args.workloads:
        N, T, L, V = CFG[name]
        U = L + 1
        assert L <= T, "every modified lattice needs a path"
        rng = np.random.default_rng(1)
        labels = torch.as_tensor(rng.integers(1, V, size=(N, L)).astype(np.int32)).to(dev)
        tl = torch.full((N,), T, dtype=torch.int32, device=dev)
        ul = torch.full((N,), L, dtype=torch.int32, device=dev)
        costs = torch.empty(N, device=dev)
        gen = torch.Generator(dev).manual_seed(7)
        opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream(dev).cuda_stream, blank_label=0,
                             maxT=T, maxU=U, batch_first=True)
        ws = torch.empty(wr.workspace_size(T, U, N, 4), dtype=torch.uint8, device=dev)
        for tag, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
            acts = torch.rand((N, T, U, V), device=dev, generator=gen).to(dt)
            grads = torch.empty_like(acts)
            out["%s_dense_%s" % (name, tag)] = compare(
                {k: (lambda k=k: wr.gpu_rnnt_async(acts, labels, tl, ul, costs, grads, 0, 1.0, ws, rnnt_type=k))
                 for k in TOPOS}, args.rounds, args.steps)
            del acts, grads
            torch.cuda.empty_cache()
        del ws
        # the joint with its ranges: forward (prepare_backward), ranges at R = 4, backward
        trans = torch.randn((N, T, V), device=dev, generator=gen)
        pred = torch.randn((N, U, V), device=dev, generator=gen)
        ranges = {k: torch.empty((N, T), dtype=torch.int32, device=dev) for k in TOPOS}
        for stag, (lm, am) in (("plain", (0.0, 0.0)), ("smoothed_0.25_0", (0.25, 0.0))):
            tt, pp = trans.clone().requires_grad_(True), pred.clone().requires_grad_(True)

            def step(k, lm=lm, am=am, tt=tt, pp=pp):
                loss, r = pruned.add_joint_rnnt_loss_with_ranges(tt, pp, labels, tl, ul, 4, reduction='sum',
                                                                 lm_only_scale=lm, am_only_scale=am, rnnt_type=k)
                loss.backward()
                ranges[k].copy_(r)
            out["%s_joint_ranges_%s" % (name, stag)] = compare({k: (lambda k=k: step(k)) for k in TOPOS},
                                                               args.rounds, args.steps)
        # pruned at R = 4 over each topology's own windows of the smoothed simple loss
        R = 4
        for k in TOPOS:
            step(k)
        torch.cuda.synchronize()
        x = torch.rand((N, T, R, V), device=dev, generator=gen)
        g = torch.empty_like(x)
        wsp = torch.empty(pruned.pruned_workspace_size(T, U, R, N, 4), dtype=torch.uint8, device=dev)

        def pstep(k):
            st = lib.rnnt_b200_pruned_loss_async_topo(0, 0, x.data_ptr(), g.data_ptr(), ranges[k].data_ptr(), R,
                                                      labels.data_ptr(), ul.data_ptr(), tl.data_ptr(), V, N,
                                                      costs.data_ptr(), 1.0, wr.rnntGradOptions(),
                                                      wr.rnntLatticeOptions(), TOPOS[k], wsp.data_ptr(), opt)
            assert st == 0, wr.status_string(st)
        out["%s_pruned_R4_fp32" % name] = compare({k: (lambda k=k: pstep(k)) for k in TOPOS}, args.rounds,
                                                  args.steps)
        pstep("modified")
        torch.cuda.synchronize()
        out["%s_pruned_R4_modified_finite_costs" % name] = int(torch.isfinite(costs).sum())   # of N
        del x, g, wsp, trans, pred
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
