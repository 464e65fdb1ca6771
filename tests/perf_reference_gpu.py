"""(Manual perf script, lives under tests/ because it executes oracle/_ref; not collected by pytest.)
Times the reference's own CUDA kernels (oracle/_ref/libwarprnnt_ref_gpu.so, compiled for sm_90)
on the BASELINE shapes — the denominator of the north-star '>= 10x the reference GPU kernel'.
Timed like tests/test_time.cu: wall clock around compute_rnnt_loss (it synchronises), 10 calls."""
import ctypes as C
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "warp-transducer_b200"))
import warprnnt_pytorch.warp_rnnt as wr  # noqa: E402
from oracle import pyoracle  # noqa: E402

CFG = {"c2": (128, 150, 40, 28), "c3": (128, 150, 20, 5000), "c4": (64, 1500, 300, 50)}


def main():
    ref = C.CDLL(pyoracle.ref_gpu_path())
    ref.compute_rnnt_loss.restype = C.c_int
    ref.compute_rnnt_loss.argtypes = [C.c_void_p] * 5 + [C.c_int, C.c_int, C.c_void_p, C.c_void_p, wr.rnntOptions]
    ref.get_workspace_size.argtypes = [C.c_int, C.c_int, C.c_int, C.c_bool, C.POINTER(C.c_size_t), C.c_size_t]
    dev = torch.device("cuda:0")
    for name in sys.argv[1:] or ["c2", "c3", "c4"]:
        N, T, L, V = CFG[name]
        U = L + 1
        acts = torch.rand((N, T, U, V), device=dev)
        grads = torch.empty_like(acts)
        labels = torch.as_tensor(np.random.default_rng(1).integers(1, V, size=(N, L)).astype(np.int32)).to(dev)
        tl = torch.full((N,), T, dtype=torch.int32, device=dev)
        ul = torch.full((N,), L, dtype=torch.int32, device=dev)
        opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream().cuda_stream,
                             blank_label=0, maxT=T, maxU=U, batch_first=True)
        for label, lib, wsz in (("reference-gpu", ref, None), ("b200", wr.lib(), wr.workspace_size(T, U, N, 4))):
            if wsz is None:
                n = C.c_size_t(0)
                lib.get_workspace_size(T, U, N, True, C.byref(n), 4)
                wsz = n.value
            ws = torch.empty(wsz, dtype=torch.uint8, device=dev)
            costs = np.zeros(N, np.float32)
            ts = []
            for it in range(13):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                st = lib.compute_rnnt_loss(acts.data_ptr(), grads.data_ptr(), labels.data_ptr(), ul.data_ptr(),
                                           tl.data_ptr(), V, N, costs.ctypes.data, ws.data_ptr(), opt)
                ts.append((time.perf_counter() - t0) * 1e3)
                assert st == 0
            t = float(np.mean(ts[3:]))
            print("%s %-13s N=%d T=%d U=%d V=%d: %.3f ms/call (10 calls, wall clock incl. sync)  %.0f utt/s  cost0=%.3f"
                  % (name, label, N, T, U, V, t, N / t * 1e3, costs[0]), flush=True)


if __name__ == "__main__":
    main()
