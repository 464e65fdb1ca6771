"""Additive-joint variant (rnnt_b200_add_joint_loss / AddJointRNNTLoss): must equal the dense path
on acts = trans[:, :, None, :] + pred[:, None, :, :] with the gradient reduced onto the factors —
checked against the fp64 oracle run on the materialised logits."""
import numpy as np
import pytest
import torch

from joint_reference import assert_joint_close, grad_mismatch, reference

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape", [(3, 9, 5, 28, 0), (2, 17, 34, 13, 4), (4, 30, 8, 300, 0),
                                   (2, 6, 3, 5000, 7), (3, 12, 1, 9, 0), (2, 1, 4, 6, 0), (5, 70, 66, 50, 0),
                                   (2, 33, 32, 130, 0),    # fused gradient kernel: 32 label positions, 2 chunks, V % 4 != 0
                                   (2, 70, 21, 520, 3),    # fused: 3 chunks, 5 vocabulary tiles (the last with 8 rows)
                                   (2, 40, 33, 64, 0),     # 33 label positions: the two-kernel gradient path
                                   (2, 6, 20, 3, 0),       # V = 3: almost every label repeats (sparse terms)
                                   (1, 1, 2, 4, 0)],
                         ids=lambda s: "N%d_T%d_U%d_V%d_b%d" % s)
def test_add_joint_matches_dense_oracle(shape):
    from warprnnt_pytorch.joint import AddJointRNNTLoss
    N, T, U, V, blank = shape
    rng = np.random.default_rng(31)
    trans = (rng.standard_normal((N, T, V)) * 2).astype(np.float32)
    pred = (rng.standard_normal((N, U, V)) * 2).astype(np.float32)
    choices = np.array([k for k in range(V) if k != blank], np.int32)
    labels = rng.choice(choices, size=(N, max(U - 1, 0))).astype(np.int32)
    tl = rng.integers(max(1, T // 2), T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0] = T, U - 1
    c_ref, df_ref, dg_ref = reference(trans, pred, labels, tl, ul, blank)
    tt = torch.tensor(trans, device="cuda", requires_grad=True)
    pp = torch.tensor(pred, device="cuda", requires_grad=True)
    lab = torch.as_tensor(labels if labels.size else np.zeros((N, 0), np.int32)).cuda()
    out = AddJointRNNTLoss(blank=blank, reduction='none')(tt, pp, lab, torch.as_tensor(tl).cuda(),
                                                          torch.as_tensor(ul).cuda())
    w = torch.linspace(0.5, 1.5, N, device="cuda")
    (out * w).sum().backward()
    assert_joint_close(out.detach().cpu().numpy(), tt.grad.cpu().numpy(), pp.grad.cpu().numpy(), c_ref, df_ref, dg_ref,
                       labels, tl, ul, blank, scale=w.cpu().numpy())


def test_add_joint_equals_dense_operator_and_reductions():
    from warprnnt_pytorch import RNNTLoss
    from warprnnt_pytorch.joint import add_joint_rnnt_loss
    rng = np.random.default_rng(32)
    N, T, U, V = 4, 20, 7, 64
    trans = torch.tensor(rng.standard_normal((N, T, V)).astype(np.float32), device="cuda", requires_grad=True)
    pred = torch.tensor(rng.standard_normal((N, U, V)).astype(np.float32), device="cuda", requires_grad=True)
    labels = torch.as_tensor(rng.integers(1, V, size=(N, U - 1)).astype(np.int32)).cuda()
    tl = torch.tensor([T, 15, 20, 11], dtype=torch.int32).cuda()
    ul = torch.tensor([U - 1, 3, 0, 6], dtype=torch.int32).cuda()
    for reduction in ("mean", "sum"):
        trans.grad = pred.grad = None
        loss = add_joint_rnnt_loss(trans, pred, labels, tl, ul, reduction=reduction)
        loss.backward()
        g1, g2 = trans.grad.clone(), pred.grad.clone()
        trans.grad = pred.grad = None
        acts = trans.unsqueeze(2) + pred.unsqueeze(1)          # the reference's way, test_time.py:73
        dense = RNNTLoss(reduction=reduction)(acts.contiguous(), labels, tl, ul)
        dense.backward()
        assert torch.allclose(loss, dense, rtol=1e-5)
        lab_np, tl_np, ul_np = labels.cpu().numpy(), tl.cpu().numpy(), ul.cpu().numpy()
        problems = grad_mismatch(g1.cpu().numpy(), trans.grad.double().cpu().numpy(), tl_np, lab_np, ul_np, 0, "dF") + \
            grad_mismatch(g2.cpu().numpy(), pred.grad.double().cpu().numpy(), ul_np + 1, lab_np, ul_np, 0, "dG")
        assert not problems, "\n".join(problems)
    with pytest.raises(ValueError):
        add_joint_rnnt_loss(trans, pred[:, :-1].contiguous(), labels, tl, ul)
    with pytest.raises(RuntimeError):
        add_joint_rnnt_loss(trans.detach().cpu(), pred.detach().cpu(), labels.cpu(), tl.cpu(), ul.cpu())
