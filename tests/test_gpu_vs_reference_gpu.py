"""Cross-check against the REFERENCE'S OWN CUDA kernels: stored outputs of the unmodified reference GPU
path (tests/golden/ref_gpu_cases.npz, written by `tests/golden/make_golden.py --ref-gpu` with the reference
compiled for sm_90 by oracle/Makefile) on fixed inputs that are recomputed here (pyoracle.REF_GPU_CASES),
including BASELINE's headline shape at full size.  Costs are compared for every utterance; gradients at
GRAD_SAMPLES seeded positions per case, and through per-utterance sums of squares over all elements.
The reference GPU path is fp32 throughout, so its own rounding noise (alpha/beta of magnitude ~1e3
carried in fp32) bounds how tight this can be; the tight parity bound is the fp64 oracle in
test_gpu_parity.py."""
import os

import numpy as np
import pytest
import torch

from oracle import pyoracle

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_gpu_cases.npz")


@pytest.fixture(scope="module")
def stored():
    return np.load(GOLDEN)


def run_ours(name):
    import warprnnt_pytorch.warp_rnnt as wr
    acts, labels, tl, ul, idx = pyoracle.ref_gpu_case_inputs(name, torch.device("cuda:0"))
    N, T, U, V = acts.shape
    costs, grads = pyoracle.gpu_loss(wr.lib(), wr.workspace_size(T, U, N, 4), acts, labels, tl, ul,
                                     wr.rnntOptions)
    del acts
    return costs, grads, idx


def rel_diff(g, gr):   # tests/test.h:22-32 metric
    g, gr = g.astype(np.float64), gr.astype(np.float64)
    return float(((g - gr) ** 2).sum() / (gr ** 2).sum())


@pytest.mark.parametrize("name", ["small", "readme_small_vocab", "readme_large_vocab_N4"])
def test_same_answers_as_reference_gpu_kernels(stored, name):
    costs, g, idx = run_ours(name)
    assert np.allclose(costs, stored[name + ".costs"], rtol=1e-5)
    assert torch.isfinite(g).all()
    at, sumsq = pyoracle.grad_summary(g, idx)
    gr = stored[name + ".grads_at"]
    assert rel_diff(at, gr) < 1e-6
    assert np.allclose(at, gr, rtol=5e-3, atol=2e-6)
    assert np.allclose(sumsq, stored[name + ".sumsq"], rtol=2e-3)


def test_headline_shape_full_size_matches_reference_gpu(stored):
    """N=128, T=150, L=20, A=5000: 2 016 000 000 gradient elements."""
    costs, g, idx = run_ours("headline")
    assert np.allclose(costs, stored["headline.costs"], rtol=1e-5)
    at, sumsq = pyoracle.grad_summary(g, idx)
    del g
    torch.cuda.empty_cache()
    gr = stored["headline.grads_at"].astype(np.float64)
    assert rel_diff(at, gr) < 1e-6
    # fp32 reference noise at |ll| ~ 1.4e3 is ~1e-3 relative; ours is far inside it
    worst = float((np.abs(at - gr) / (2e-6 + 1e-2 * np.abs(gr))).max())
    assert worst <= 1.0, worst
    assert np.allclose(sumsq, stored["headline.sumsq"], rtol=2e-3)
