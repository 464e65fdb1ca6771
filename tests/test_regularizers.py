"""Gradient options (FastEmit, clamp) without a GPU: the fp64 reference the GPU tests compare against,
derived independently with torch autograd, and the C-ABI / Python argument rules, which are checked
before any device access."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import pyoracle
from regularized_reference import rnnt_logits_reg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make_case(seed, N, T, U, V, blank):
    rng = np.random.default_rng(seed)
    acts = rng.standard_normal((N, T, U, V)) * 2
    choices = np.array([k for k in range(V) if k != blank], np.int32)
    labels = rng.choice(choices, size=(N, U - 1)).astype(np.int32)
    tl = rng.integers(1, T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0] = T, U - 1
    tl[-1], ul[-1] = 1, 0          # T == 1 and U == 1 in one utterance
    if N > 2:
        ul[1] = 0                  # U == 1 with T > 1
    return acts, labels, tl, ul


def surrogate_grad(acts, labels, tl, ul, blank, lam):
    """d/dx of  sum_b [ -ll_b - lam * sum_{t,u} sg[e_y(t,u)] * lp_y(t,u) ]  by torch fp64 autograd, with a
    lattice written out here (independent of the oracle)."""
    x = torch.tensor(acts, dtype=torch.float64, requires_grad=True)
    total = x.new_zeros(())
    for b in range(x.shape[0]):
        T, U = int(tl[b]), int(ul[b]) + 1
        lp = torch.log_softmax(x[b, :T, :U], dim=-1)
        lpb = lp[..., blank]
        y = torch.as_tensor(labels[b, :U - 1], dtype=torch.long)
        lpy = lp[:, :U - 1].gather(2, y.view(1, -1, 1).expand(T, U - 1, 1))[..., 0]
        alpha = [[None] * U for _ in range(T)]
        for t in range(T):
            for u in range(U):
                terms = []
                if t > 0:
                    terms.append(alpha[t - 1][u] + lpb[t - 1, u])
                if u > 0:
                    terms.append(alpha[t][u - 1] + lpy[t, u - 1])
                alpha[t][u] = torch.logsumexp(torch.stack(terms), 0) if terms else x.new_zeros(())
        ll = alpha[T - 1][U - 1] + lpb[T - 1, U - 1]
        with torch.no_grad():
            beta = [[None] * U for _ in range(T)]
            for t in range(T - 1, -1, -1):
                for u in range(U - 1, -1, -1):
                    if t == T - 1 and u == U - 1:
                        beta[t][u] = lpb[t, u]
                        continue
                    terms = []
                    if t < T - 1:
                        terms.append(beta[t + 1][u] + lpb[t, u])
                    if u < U - 1:
                        terms.append(beta[t][u + 1] + lpy[t, u])
                    beta[t][u] = torch.logsumexp(torch.stack(terms), 0)
            e_y = torch.zeros(T, max(U - 1, 0), dtype=torch.float64)
            for t in range(T):
                for u in range(U - 1):
                    e_y[t, u] = torch.exp(alpha[t][u] + lpy[t, u] + beta[t][u + 1] - ll)
        total = total - ll - lam * (e_y * lpy).sum()
    total.backward()
    return x.grad.numpy()


@pytest.mark.parametrize("case", [(1, 4, 6, 4, 7, 2), (2, 3, 5, 3, 5, 4), (3, 5, 4, 5, 6, 0)],
                         ids=lambda c: "seed%d_N%d_T%d_U%d_V%d_b%d" % c)
@pytest.mark.parametrize("lam", [0.01, 0.5, 2.0])
def test_fastemit_reference_matches_autograd_of_the_surrogate(case, lam):
    seed, N, T, U, V, blank = case
    acts, labels, tl, ul = make_case(seed, N, T, U, V, blank)
    c_ref, g_ref = rnnt_logits_reg(acts, labels, tl, ul, blank, fastemit_lambda=lam)
    g_auto = surrogate_grad(acts, labels, tl, ul, blank, lam)
    assert np.abs(g_ref - g_auto).max() < 1e-10, np.abs(g_ref - g_auto).max()
    c0, g0, _ = pyoracle.rnnt_logits(acts, labels, tl, ul, blank)
    assert np.array_equal(c_ref, c0)                      # costs do not depend on the options
    assert np.abs(g_ref - g0).max() > 1e-3 * lam           # and FastEmit does move the gradient
    for b in range(N):                                     # padded cells stay exact zeros
        assert not g_ref[b, tl[b]:].any() and not g_ref[b, :, ul[b] + 1:].any()


def test_reference_without_options_is_the_oracle_and_clamp_is_a_clip():
    acts, labels, tl, ul = make_case(4, 4, 6, 4, 9, 3)
    c0, g0, _ = pyoracle.rnnt_logits(acts, labels, tl, ul, 3)
    c, g = rnnt_logits_reg(acts, labels, tl, ul, 3)
    assert np.array_equal(c, c0) and np.array_equal(g, g0)
    clip = float(np.quantile(np.abs(g0[g0 != 0]), 0.9))
    c, g = rnnt_logits_reg(acts, labels, tl, ul, 3, clamp=clip)
    assert np.array_equal(c, c0) and np.array_equal(g, np.clip(g0, -clip, clip))
    assert (np.abs(g0) > clip).mean() > 0.01
    _, g_fe = rnnt_logits_reg(acts, labels, tl, ul, 3, fastemit_lambda=0.5)
    _, g_both = rnnt_logits_reg(acts, labels, tl, ul, 3, fastemit_lambda=0.5, clamp=clip)
    assert np.array_equal(g_both, np.clip(g_fe, -clip, clip))


# ------------------------------------------------------------------ C-ABI and Python argument rules
@pytest.fixture(scope="module")
def wr():
    import warprnnt_pytorch.warp_rnnt as wr
    return wr


def test_new_entries_are_exported_and_codes_pinned(wr, tmp_path):
    out = subprocess.run(["nm", "-D", "--defined-only", wr.lib_path()], capture_output=True, text=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    for s in ("rnnt_b200_loss_async_ex", "rnnt_b200_backward_ex", "rnnt_b200_add_joint_backward_ex"):
        assert s in exported, s
    assert (wr.RNNT_B200_FP32, wr.RNNT_B200_BF16, wr.RNNT_B200_FP16, wr.RNNT_B200_FP64) == (0, 1, 2, 3)
    assert C.sizeof(wr.rnntGradOptions) == 8 and C.sizeof(wr.rnntOptions) == 32
    src = tmp_path / "codes.c"
    src.write_text('#include "rnnt.h"\n'
                   '_Static_assert(RNNT_B200_FP32 == 0 && RNNT_B200_BF16 == 1 && RNNT_B200_FP16 == 2 && '
                   'RNNT_B200_FP64 == 3, "dtype codes");\n'
                   '_Static_assert(sizeof(struct rnntGradOptions) == 8 && sizeof(struct rnntOptions) == 32, "sizes");\n'
                   'int main(void) { return 0; }\n')
    subprocess.check_call(["/usr/bin/gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-c",
                           "-o", str(tmp_path / "codes.o")])


BAD_OPTIONS = [(-0.1, 0.0), (float("nan"), 0.0), (float("inf"), 0.0), (-float("inf"), 0.0), (0.0, float("nan")),
               (0.5, float("nan"))]


def test_invalid_options_are_rejected_before_device_access(wr):
    """Every call here returns INVALID_VALUE (2) from the argument checks, before any CUDA call; the
    buffers are host memory and are never dereferenced."""
    lib = wr.lib()
    buf = (C.c_float * 256)()
    ibuf = (C.c_int * 8)(1, 1, 1, 1, 1, 1, 1, 1)
    p, ip = C.addressof(buf), C.addressof(ibuf)
    opt = wr.rnntOptions(loc=1, num_threads=0, stream=None, blank_label=0, maxT=2, maxU=2, batch_first=True)
    for lam, clamp in BAD_OPTIONS:
        g = wr.rnntGradOptions(lam, clamp)
        for code in (0, 1, 2, 3):
            assert lib.rnnt_b200_loss_async_ex(code, 0, p, p, ip, ip, ip, 4, 1, p, 1.0, g, p, opt) == 2
            assert lib.rnnt_b200_backward_ex(code, p, p, ip, ip, ip, 4, 1, None, 1.0, g, p, opt) == 2
    lib.rnnt_b200_add_joint_backward_ex.restype = C.c_int
    lib.rnnt_b200_add_joint_backward_ex.argtypes = [C.c_void_p] * 7 + [C.c_int, C.c_int, C.c_void_p, C.c_float,
                                                                         wr.rnntGradOptions, C.c_void_p, wr.rnntOptions]
    for lam, clamp in BAD_OPTIONS + [(0.0, 1.0), (0.3, 0.5), (0.0, -1.0)]:   # the joint takes no clamp at all
        g = wr.rnntGradOptions(lam, clamp)
        assert lib.rnnt_b200_add_joint_backward_ex(p, p, p, p, ip, ip, ip, 4, 1, None, 1.0, g, p, opt) == 2
    good = wr.rnntGradOptions(0.5, 1.0)
    # unknown dtype / layout, and the 16-bit time-major combination no plain entry offers
    assert lib.rnnt_b200_loss_async_ex(4, 0, p, p, ip, ip, ip, 4, 1, p, 1.0, good, p, opt) == 2
    assert lib.rnnt_b200_loss_async_ex(0, 2, p, p, ip, ip, ip, 4, 1, p, 1.0, good, p, opt) == 2
    assert lib.rnnt_b200_loss_async_ex(1, 1, p, p, ip, ip, ip, 4, 1, p, 1.0, good, p, opt) == 2
    assert lib.rnnt_b200_backward_ex(7, p, p, ip, ip, ip, 4, 1, None, 1.0, good, p, opt) == 2
    # valid options still go through the ordinary argument checks
    assert lib.rnnt_b200_loss_async_ex(0, 0, None, p, ip, ip, ip, 4, 1, p, 1.0, good, p, opt) == 2
    assert lib.rnnt_b200_backward_ex(0, p, None, ip, ip, ip, 4, 1, None, 1.0, good, p, opt) == 2


def test_python_options_are_validated():
    from warprnnt_pytorch import RNNTLoss, rnnt_loss, warp_rnnt
    from warprnnt_pytorch.distributed import ShardedRNNTLoss
    from warprnnt_pytorch.joint import AddJointRNNTLoss, add_joint_rnnt_loss
    for lam, clamp in BAD_OPTIONS + [(1e39, 0.0)]:
        with pytest.raises(ValueError):
            RNNTLoss(fastemit_lambda=lam, clamp=clamp)
        with pytest.raises(ValueError):
            ShardedRNNTLoss(fastemit_lambda=lam, clamp=clamp)
        with pytest.raises(ValueError):
            warp_rnnt.grad_options(lam, clamp)
    acts = torch.zeros(1, 2, 3, 5)
    labels = torch.tensor([[1, 2]], dtype=torch.int32)
    tl, ul = torch.tensor([2], dtype=torch.int32), torch.tensor([2], dtype=torch.int32)
    with pytest.raises(ValueError):          # before the operator looks at the device
        rnnt_loss(acts, labels, tl, ul, fastemit_lambda=-1.0)
    with pytest.raises(RuntimeError):        # valid options: the usual no-CPU-fallback error
        rnnt_loss(acts, labels, tl, ul, fastemit_lambda=0.1, clamp=1.0)
    with pytest.raises(TypeError):           # keyword-only: the reference's positional signature is unchanged
        RNNTLoss(0, 'mean', 0.1)
    assert warp_rnnt.grad_options() is None and warp_rnnt.grad_options(0.0, 0.0) is None
    g = warp_rnnt.grad_options(0.25, 2.0)
    assert (g.fastemit_lambda, g.clamp) == (0.25, 2.0)
    assert warp_rnnt.grad_options(0.0, 3.0).clamp == 3.0
    with pytest.raises(ValueError, match="additive joint"):
        AddJointRNNTLoss(clamp=1.0)
    with pytest.raises(ValueError, match="additive joint"):
        add_joint_rnnt_loss(torch.zeros(1, 2, 5), torch.zeros(1, 3, 5), labels, tl, ul, clamp=-1.0)
    with pytest.raises(ValueError):
        AddJointRNNTLoss(fastemit_lambda=math.nan)
    AddJointRNNTLoss(fastemit_lambda=0.3)
