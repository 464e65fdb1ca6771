#!/usr/bin/env python
"""Regenerates the committed golden fixtures from the reference implementation (needs the reference
sources, $RNNT_REFERENCE, and oracle/_ref built from them by oracle/Makefile); the test suite reads the
committed outputs, never the reference.

    python tests/golden/make_golden.py                 # known_answers.json, ref_cases.npz, ref_live_cpu.npz
    python tests/golden/make_golden.py --ref-gpu DIR   # DIR/ref_gpu_cases.npz (needs a GPU and
                                                       # oracle/_ref/libwarprnnt_ref_gpu.so only)

Outputs (next to this script):
  known_answers.json  the known-answer vectors the reference's own tests hold for this path,
                      extracted mechanically from the reference test sources (citations inside)
  ref_cases.npz       seeded random cases (incl. ragged lengths, blank != 0, U == 1, V % 4 != 0)
                      with the outputs of the REFERENCE ITSELF:
                        - oracle/_ref/libwarprnnt_ref_cpu.so (compiled unmodified reference CPU
                          path) composed with log_softmax fwd/bwd, fp32 and fp64
                        - pytorch_binding/test/transducer_np.py (the reference's numpy model)
  ref_live_cpu.npz    the reference CPU library itself (log-prob and logits conventions, with and
                      without gradients) on the seeded cases of tests/test_oracle.py
  ref_gpu_cases.npz   the reference's own CUDA kernels on the fixed inputs of pyoracle.REF_GPU_CASES:
                      costs, gradients at GRAD_SAMPLES seeded positions, per-utterance sums of squares
"""
import importlib.util
import json
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("RNNT_REFERENCE", "/root/reference")
sys.path.insert(0, ROOT)
from oracle import pyoracle  # noqa: E402


def cxx_vector(src, func, name):
    """Pull `std::vector<...> name = {...};` out of function `func` in a C++ test source."""
    body = src[src.index("bool %s()" % func):]
    m = re.search(r"std::vector<\w+>\s+%s\s*=\s*\{([^}]*)\}" % name, body)
    return [float(x) for x in m.group(1).replace("\n", " ").split(",") if x.strip()]


def known_answers():
    cpu = open(os.path.join(REF, "tests/test_cpu.cpp")).read()
    gpu = open(os.path.join(REF, "tests/test_gpu.cu")).read()
    out = {
        "_source": "extracted from the reference test-suite by tests/golden/make_golden.py",
        "small": {
            "cite": ["tests/test_cpu.cpp:12-71", "tests/test_gpu.cu:18-94",
                     "pytorch_binding/test/test.py:51-78"],
            "shape": [1, 2, 3, 5], "labels": [[1, 2]], "blank": 0,
            "acts": cxx_vector(gpu, "small_test", "acts"),
            "cost": 4.495666, "cost_tol_abs": 1e-4,
        },
        "options": {
            "cite": ["tests/test_cpu.cpp:73-179", "tests/test_gpu.cu:96-224",
                     "pytorch_binding/test/test.py:80-161",
                     "tensorflow_binding/tests/test_warprnnt_op.py:54-85"],
            "shape": [2, 4, 3, 3], "labels": [[1, 2], [1, 1]], "blank": 0,
            "acts": cxx_vector(gpu, "options_test", "acts"),
            "costs": [4.2806528590890736, 3.9384369822503591],
            "logits_grads": cxx_vector(gpu, "options_test", "expected_grads"),
            "logprob_grads": cxx_vector(cpu, "options_test", "expected_grads"),
            "tol_abs": 1e-4,
        },
    }
    assert out["options"]["acts"] == cxx_vector(cpu, "options_test", "acts")
    assert len(out["small"]["acts"]) == 30 and len(out["options"]["logits_grads"]) == 72
    # the 30 logits-gradients of the small case live in the PyTorch test (test.py:62-74)
    py = open(os.path.join(REF, "pytorch_binding/test/test.py")).read()
    seg = py[py.index("def small_test"):py.index("def big_test")]
    m = re.search(r"expected_grads = np\.array\((.*?)\)\n", seg, re.S)
    out["small"]["logits_grads"] = np.array(eval(m.group(1))).reshape(-1).tolist()
    seg = py[py.index("def big_test"):]
    m = re.search(r"activations = (\[.*?\]\]\]\])", seg, re.S)
    out["options"]["acts_f64"] = np.array(eval(m.group(1))).reshape(-1).tolist()
    m = re.search(r"expected_grads = (\[.*?\]\]\]\])", seg, re.S)
    out["options"]["logits_grads_hi"] = np.array(eval(m.group(1))).reshape(-1).tolist()
    return out


def load_transducer_np():
    path = os.path.join(REF, "pytorch_binding/test/transducer_np.py")
    spec = importlib.util.spec_from_file_location("transducer_np", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


CASES = [
    # name, N, T, U, V, blank, ragged, scale
    ("full_small", 3, 6, 4, 8, 0, False, 1.0),
    ("ragged", 4, 9, 5, 7, 0, True, 1.0),
    ("blank_last", 2, 7, 4, 6, 5, True, 1.0),
    ("blank_mid", 2, 5, 6, 9, 3, True, 2.0),
    ("u1_empty_labels", 2, 6, 1, 5, 0, True, 1.0),
    ("t1", 2, 1, 4, 5, 0, False, 1.0),
    ("v_odd", 2, 8, 5, 13, 0, True, 3.0),
    ("v_wide", 1, 5, 3, 301, 0, False, 4.0),
    ("u_gt_32", 1, 12, 40, 6, 0, False, 1.0),
    ("big_range", 2, 6, 4, 10, 0, True, 30.0),
]


def make_case(rng, N, T, U, V, blank, ragged, scale):
    acts = (rng.standard_normal((N, T, U, V)) * scale).astype(np.float32)
    choices = [k for k in range(V) if k != blank]
    labels = rng.choice(choices, size=(N, max(U - 1, 0))).astype(np.int32)
    if ragged and N > 1:
        act_lens = rng.integers(max(1, T // 2), T + 1, size=N).astype(np.int32)
        label_lens = rng.integers(0, U, size=N).astype(np.int32)
        act_lens[0] = T           # certify_inputs requires max(len) == dim
        label_lens[0] = U - 1
    else:
        act_lens = np.full(N, T, np.int32)
        label_lens = np.full(N, U - 1, np.int32)
    return acts, labels, act_lens, label_lens


LIVE_CPU_SHAPES = [(3, 11, 6, 10), (2, 50, 10, 15), (65, 10, 5, 5), (1, 50, 15, 20)]
LIVE_CPU_SAMPLES = 256


def live_cpu_case(i, rng):
    """Case i of tests/test_oracle.py::test_against_reference_cpu_library (draws from the shared rng)."""
    N, T, U, V = LIVE_CPU_SHAPES[i]
    acts = rng.random((N, T, U, V), dtype=np.float32)      # U[0,1) like tests/random.cpp:13-20
    labels = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    tl = rng.integers(T // 2 + 1, T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0] = T, U - 1
    idx = np.sort(np.random.default_rng(100 + i).integers(0, acts.size, size=LIVE_CPU_SAMPLES))
    return acts, labels, tl, ul, idx


def live_cpu():
    rng = np.random.default_rng(7)
    blob = {}
    for i in range(len(LIVE_CPU_SHAPES)):
        acts, labels, tl, ul, idx = live_cpu_case(i, rng)
        lp = pyoracle.log_softmax_np(acts)
        c_ref, g_ref = pyoracle.ref_cpu_logprobs(lp, labels, tl, ul, 0, threads=2)
        c_fwd, _ = pyoracle.ref_cpu_logprobs(lp, labels, tl, ul, 0, want_grad=False)
        c64, dx64 = pyoracle.ref_cpu_logits(acts.astype(np.float64), labels, tl, ul, 0)
        blob.update({"%d.costs" % i: c_ref, "%d.grads_at" % i: g_ref.reshape(-1)[idx],
                     "%d.costs_fwd" % i: c_fwd, "%d.costs_f64" % i: c64,
                     "%d.dx_f64_at" % i: dx64.reshape(-1)[idx]})
    np.savez_compressed(os.path.join(HERE, "ref_live_cpu.npz"), **blob)


def ref_gpu(out_dir):
    """The reference's CUDA kernels (oracle/_ref/libwarprnnt_ref_gpu.so) on pyoracle.REF_GPU_CASES."""
    import ctypes as C
    import torch
    ref = C.CDLL(pyoracle.ref_gpu_path())
    ref.compute_rnnt_loss.restype = C.c_int
    ref.compute_rnnt_loss.argtypes = [C.c_void_p] * 5 + [C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                                         pyoracle.RnntOptions]
    ref.get_workspace_size.argtypes = [C.c_int, C.c_int, C.c_int, C.c_bool, C.POINTER(C.c_size_t), C.c_size_t]
    dev = torch.device("cuda:0")
    blob = {"names": np.array(sorted(pyoracle.REF_GPU_CASES))}
    for name in sorted(pyoracle.REF_GPU_CASES):
        acts, labels, tl, ul, idx = pyoracle.ref_gpu_case_inputs(name, dev)
        N, T, U, V = acts.shape
        n = C.c_size_t(0)
        assert ref.get_workspace_size(T, U, N, True, C.byref(n), 4) == 0
        costs, grads = pyoracle.gpu_loss(ref, n.value, acts, labels, tl, ul, pyoracle.RnntOptions)
        at, sumsq = pyoracle.grad_summary(grads, idx)
        blob.update({name + ".costs": costs, name + ".grads_at": at, name + ".sumsq": sumsq})
        print("%-22s N=%d T=%d U=%d V=%d cost0=%.4f" % (name, N, T, U, V, costs[0]), flush=True)
        del acts, grads
        torch.cuda.empty_cache()
    os.makedirs(out_dir, exist_ok=True)
    np.savez_compressed(os.path.join(out_dir, "ref_gpu_cases.npz"), **blob)


def main():
    if "--ref-gpu" in sys.argv:
        return ref_gpu(sys.argv[sys.argv.index("--ref-gpu") + 1])
    if not os.path.isdir(REF):
        sys.exit("reference sources not found (set RNNT_REFERENCE)")
    pyoracle.build()
    assert pyoracle.have_ref_cpu()
    json.dump(known_answers(), open(os.path.join(HERE, "known_answers.json"), "w"), indent=1)

    tnp = load_transducer_np()
    rng = np.random.default_rng(20260924)
    blob = {"names": np.array([c[0] for c in CASES])}
    for name, N, T, U, V, blank, ragged, scale in CASES:
        acts, labels, act_lens, label_lens = make_case(rng, N, T, U, V, blank, ragged, scale)
        c32, g32 = pyoracle.ref_cpu_logits(acts, labels, act_lens, label_lens, blank, threads=1)
        c64, g64 = pyoracle.ref_cpu_logits(acts.astype(np.float64), labels, act_lens, label_lens,
                                           blank, threads=1)
        # the reference's numpy model (log-prob gradient convention) on the same log-probs
        lp = pyoracle.log_softmax_np(acts.astype(np.float64))
        if U > 1:
            cn, gn = tnp.transduce_batch(lp, labels, act_lens, label_lens, blank)
            gn = gn - np.exp(lp) * gn.sum(-1, keepdims=True)
        else:   # transducer_np indexes labels[u-1]; U == 1 is outside what it supports
            cn, gn = c64, g64
        assert np.allclose(cn, c64, rtol=1e-5, atol=1e-5), (name, cn, c64)
        assert np.allclose(gn, g64, rtol=1e-4, atol=1e-5), name
        blob.update({
            name + ".acts": acts, name + ".labels": labels, name + ".act_lens": act_lens,
            name + ".label_lens": label_lens, name + ".blank": np.int32(blank),
            name + ".ref_costs_f32": c32, name + ".ref_grads_f32": g32,
            name + ".ref_costs_f64": c64, name + ".ref_grads_f64": g64,
            name + ".np_costs": np.asarray(cn, np.float64),
        })
        print("%-16s N=%d T=%d U=%d V=%d blank=%d costs=%s" % (name, N, T, U, V, blank, c64))
    np.savez_compressed(os.path.join(HERE, "ref_cases.npz"), **blob)
    live_cpu()
    print("wrote", os.path.join(HERE, "known_answers.json"), os.path.join(HERE, "ref_cases.npz"))


if __name__ == "__main__":
    main()
