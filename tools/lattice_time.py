"""Device time of the loss, gradient and alignment on caller-supplied factors (DESIGN.md §13) at the lattice shapes of
the bench's C2, C3 and C4 (dev tool, not the bench).  Per workload, in one process, interleaved round by round in a
rotating order:
  lattice_step    rnnt_b200_lattice_forward (prepare_backward = 1) + rnnt_b200_lattice_backward: import, both
                  wavefronts, gradient kernel
  lattice_align   rnnt_b200_lattice_align: import, Viterbi wavefront and backtrace
  lattice_alpha   rnnt_b200_lattice_forward (prepare_backward = 0): import, alpha wavefront
  rnnt_step       for context: rnnt_b200_forward_topo (prepare_backward = 1) + rnnt_b200_backward_topo on the logits
                  [N, T, S+1, V] of the same lattice
  rnnt_alpha      for context: rnnt_b200_forward_topo with prepare_backward = 0 (pass 1 and the alpha wavefront)

    python tools/lattice_time.py [--rounds 7] [--steps 10] [--profile] [c2 c3 c4]

Prints one JSON line: the GPU, its power limit, and per workload the median ms per call of each over the rounds.
--profile adds, from a separate torch.profiler run of each workload, the mean device time of every kernel each call
launches.
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
from align_time import kernel_ms  # noqa: E402
from delay_time import power_limit_w, step_ms  # noqa: E402

# name -> (N, T, S = max label length, V of the logits the rnnt_loss context calls read)
WORKLOADS = {
    "c2": (128, 150, 40, 28),
    "c3": (128, 150, 20, 5000),
    "c4": (64, 1500, 300, 50),
}


def calls(name, dev):
    N, T, S, V = WORKLOADS[name]
    U = S + 1
    rng = np.random.default_rng(1)
    gen = torch.Generator(dev).manual_seed(7)
    lp = torch.log_softmax(torch.rand((N, U, T, 3), device=dev, generator=gen) * 3.0, -1)
    py, px = lp[..., 0].contiguous(), lp[:, :S, :, 1].contiguous()
    gx, gy = torch.empty_like(px), torch.empty_like(py)
    labels = torch.as_tensor(rng.integers(1, V, size=(N, S)).astype(np.int32)).to(dev)
    tl = torch.full((N,), T, dtype=torch.int32, device=dev)
    ul = torch.full((N,), S, dtype=torch.int32, device=dev)
    costs = torch.empty(N, device=dev)
    scores = torch.empty(N, device=dev)
    frames = torch.empty((N, S), dtype=torch.int32, device=dev)
    opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream(dev).cuda_stream, blank_label=0,
                         maxT=T, maxU=U, batch_first=True)
    lib, code = wr.lib(), wr.RNNT_B200_FP32
    lws = torch.empty(wr.lattice_workspace_size(T, U, N), dtype=torch.uint8, device=dev)
    acts = torch.rand((N, T, U, V), device=dev, generator=gen)
    grads = torch.empty_like(acts)
    ws = torch.empty(wr.workspace_size(T, U, N, 4), dtype=torch.uint8, device=dev)

    def ok(st):
        assert st == 0, wr.status_string(st)

    def lattice_forward(prep):
        ok(lib.rnnt_b200_lattice_forward(code, px.data_ptr(), py.data_ptr(), ul.data_ptr(), tl.data_ptr(), N, 0,
                                         costs.data_ptr(), prep, lws.data_ptr(), opt))

    def lattice_step():
        lattice_forward(1)
        ok(lib.rnnt_b200_lattice_backward(code, gx.data_ptr(), gy.data_ptr(), ul.data_ptr(), tl.data_ptr(), N, 0,
                                          None, 1.0, lws.data_ptr(), opt))

    def lattice_align():
        ok(lib.rnnt_b200_lattice_align(code, px.data_ptr(), py.data_ptr(), ul.data_ptr(), tl.data_ptr(), N, 0,
                                       frames.data_ptr(), scores.data_ptr(), lws.data_ptr(), opt))

    def rnnt_forward(prep):
        ok(lib.rnnt_b200_forward_topo(code, acts.data_ptr(), labels.data_ptr(), ul.data_ptr(), tl.data_ptr(), V, N,
                                      costs.data_ptr(), prep, wr.rnntLatticeOptions(), 0, ws.data_ptr(), opt))

    def rnnt_step():
        rnnt_forward(1)
        ok(lib.rnnt_b200_backward_topo(code, acts.data_ptr(), grads.data_ptr(), labels.data_ptr(), ul.data_ptr(),
                                       tl.data_ptr(), V, N, None, 1.0, wr.rnntGradOptions(), wr.rnntLatticeOptions(),
                                       0, ws.data_ptr(), opt))

    return {"lattice_step": lattice_step, "lattice_align": lattice_align,
            "lattice_alpha": lambda: lattice_forward(0), "rnnt_step": rnnt_step, "rnnt_alpha": lambda: rnnt_forward(0)}


def compare(fns, rounds, steps):
    names = list(fns)
    ms = {k: [] for k in names}
    for r in range(rounds):
        for k in names[r % len(names):] + names[:r % len(names)]:
            ms[k].append(step_ms(fns[k], steps))
    return {"ms_per_call": {k: float(np.median(v)) for k, v in ms.items()}, "all_ms": ms}


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
        fns = calls(name, dev)
        res = compare(fns, args.rounds, args.steps)
        if args.profile:
            res["kernel_ms"] = kernel_ms(fns, args.steps)
        out[name] = res
        del fns
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
