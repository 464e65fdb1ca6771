"""Child process of test_gpu_modified.py: the modified topology under one tuning-hook setting (RNNT_B200_*
environment variables, already set in this process's environment; a hook is read once per process).

    python tests/modified_hook_child.py hooks     the dense, pruned and joint shapes of hook_cases.py with
                                                  rnnt_type='modified', each against tests/modified_reference.py,
                                                  and the kernels they ran
    python tests/modified_hook_child.py groups    a grouped full call (RNNT_B200_GROUPS=4) against the forward /
                                                  backward split, which never groups: bitwise

Utterance 0 of every shape keeps U_b = U, so where U - 1 > T it has no path; the others are cut to at most T_b
labels.  Prints one JSON line {"problems": [...], "kernels": [...], "launches": {...}} ("hooks") or "groups ok".
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, os.path.join(ROOT, "warp-transducer_b200"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import hook_cases as hc  # noqa: E402
import modified_reference as mr  # noqa: E402
from joint_reference import grad_mismatch  # noqa: E402

LAM = 0.25   # delay penalty of the dense calls (exact in float32)
MOD = 1      # RNNT_B200_RNNT_MODIFIED


def cuda(*xs):
    return [torch.as_tensor(x).cuda() for x in xs]


def inputs(name, shape, joint, pruned=False):
    x, labels, tl, ul = hc.inputs(name, shape, joint, pruned)
    ul[1:] = np.minimum(ul[1:], tl[1:])
    return x, labels, tl, ul


def close(costs, grads, c_ref, g_ref, tl, ul, lam):
    problems = []
    bar = 1e-5 * np.maximum(np.abs(c_ref), 1.0 + lam * tl * (ul + 1) / 2.0)
    fin = np.isfinite(c_ref)
    if not (np.array_equal(np.isfinite(costs), fin) and (np.abs(costs[fin] - c_ref[fin]) <= bar[fin]).all()):
        problems.append("costs: %s against %s" % (costs.tolist(), c_ref.tolist()))
    if np.isnan(grads).any() or not (np.abs(grads - g_ref) <= 1e-4 * np.abs(g_ref) + 1e-6).all():
        problems.append("grads: max |err| %.3g" % np.nanmax(np.abs(grads - g_ref)))
    if grads[~fin].any():
        problems.append("an utterance without a path has a gradient")
    return problems


def dense(wr, name, shape):
    acts, labels, tl, ul = inputs(name, shape, False)
    a, lab, tld, uld = cuda(acts, labels, tl, ul)
    costs = torch.empty(shape[0], device="cuda")
    grads = torch.full_like(a, float("nan"))
    ws = wr.gpu_rnnt_async(a, lab, tld, uld, costs, grads, 0, delay_penalty=LAM, rnnt_type='modified')
    launches = wr.last_launch_count()
    torch.cuda.synchronize()
    del ws
    got = costs.cpu().numpy(), grads.cpu().numpy()

    def check():
        c_ref, g_ref = mr.dense_loss(acts, labels, tl, ul, delay_penalty=LAM)
        return close(*got, c_ref, g_ref, tl, ul, LAM)
    return check, launches


def pruned(wr, name, shape):
    from warprnnt_pytorch.pruned import pruned_workspace_size
    (logits, ranges), labels, tl, ul = inputs(name, shape, False, True)
    N, T, R, V = logits.shape
    U = shape[2]
    x, rg, lab, tld, uld = cuda(logits, ranges, labels, tl, ul)
    costs = torch.empty(N, device="cuda")
    grads = torch.full_like(x, float("nan"))
    ws = torch.empty(pruned_workspace_size(T, U, R, N, 4), dtype=torch.uint8, device="cuda")
    opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream().cuda_stream, blank_label=0,
                         maxT=T, maxU=U, batch_first=True)
    st = wr.lib().rnnt_b200_pruned_loss_async_topo(0, 0, x.data_ptr(), grads.data_ptr(), rg.data_ptr(), R,
                                                   lab.data_ptr(), uld.data_ptr(), tld.data_ptr(), V, N,
                                                   costs.data_ptr(), 1.0, wr.rnntGradOptions(0.0, 0.0),
                                                   wr.rnntLatticeOptions(0.0), MOD, ws.data_ptr(), opt)
    assert st == 0, wr.status_string(st)
    launches = wr.last_launch_count()
    torch.cuda.synchronize()
    del ws
    got = costs.cpu().numpy(), grads.cpu().numpy()

    def check():
        c_ref, g_ref = mr.loss(logits, labels, tl, ul, ranges)
        return close(*got, c_ref, g_ref, tl, ul, 0.0)
    return check, launches


def joint(wr, name, shape):
    from warprnnt_pytorch.joint import add_joint_rnnt_loss
    (trans, pred), labels, tl, ul = inputs(name, shape, True)
    tt = torch.tensor(trans, device="cuda", requires_grad=True)
    pp = torch.tensor(pred, device="cuda", requires_grad=True)
    lab, tld, uld = cuda(labels, tl, ul)
    out = add_joint_rnnt_loss(tt, pp, lab, tld, uld, 0, 'none', rnnt_type='modified')
    out[torch.isfinite(out)].sum().backward()
    launches = wr.last_launch_count()
    torch.cuda.synchronize()
    costs, dF, dG = out.detach().cpu().numpy(), tt.grad.cpu().numpy(), pp.grad.cpu().numpy()

    def check():
        c_ref, dF_ref, dG_ref = mr.joint_reference(trans.astype(np.float64), pred.astype(np.float64), labels, tl, ul)
        problems = []
        fin = np.isfinite(c_ref)
        if not (np.array_equal(np.isfinite(costs), fin) and
                (np.abs(costs[fin] - c_ref[fin]) <= 1e-5 * np.maximum(np.abs(c_ref[fin]), 1.0)).all()):
            problems.append("costs: %s against %s" % (costs.tolist(), c_ref.tolist()))
        problems += grad_mismatch(dF, dF_ref, tl, labels, ul, 0, "dF")
        problems += grad_mismatch(dG, dG_ref, ul + 1, labels, ul, 0, "dG")
        return problems
    return check, launches


def hooks():
    import warprnnt_pytorch.pruned  # noqa: F401  (argtypes of the pruned entries)
    import warprnnt_pytorch.warp_rnnt as wr
    problems, kernels, launches = [], set(), {}
    for suite, shapes, run in (("dense", hc.DENSE, dense), ("pruned", hc.DENSE, pruned), ("joint", hc.JOINT, joint)):
        for name, shape in shapes.items():
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                check, n = run(wr, name, shape)
            kernels.update(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
            problems += ["%s %s: %s" % (suite, name, q) for q in check()]   # the reference runs unprofiled
            launches["%s %s" % (suite, name)] = n
    print(json.dumps({"problems": problems, "kernels": sorted(kernels), "launches": launches}))


def groups():
    import warprnnt_pytorch.warp_rnnt as wr
    assert os.environ.get("RNNT_B200_GROUPS") == "4"
    N, T, U, V = 10, 12, 6, 28
    acts, labels, tl, ul = inputs("V28_chunk", (N, T, U, V), False)
    tl[3], ul[3] = 2, 5      # one utterance without a path
    for storage in (torch.float32, torch.float64, torch.bfloat16, torch.float16):
        a = torch.tensor(acts, device="cuda").to(storage)
        lab, tld, uld = cuda(labels, tl, ul)
        costs = torch.empty(N, device="cuda", dtype=wr.costs_dtype(a))
        grads = torch.full_like(a, float("nan"))
        ws = wr.gpu_rnnt_async(a, lab, tld, uld, costs, grads, 0, delay_penalty=LAM, rnnt_type='modified')
        assert wr.last_launch_count() == 12, wr.last_launch_count()     # 4 groups x (pass 1, lattice, pass 2)
        c2 = torch.empty_like(costs)
        ws2 = wr.gpu_rnnt_forward(a, lab, tld, uld, c2, 0, delay_penalty=LAM, rnnt_type='modified')
        assert wr.last_launch_count() == 2
        g2 = torch.full_like(a, float("nan"))
        wr.gpu_rnnt_backward(a, lab, tld, uld, g2, None, 0, 1.0, ws2, delay_penalty=LAM, rnnt_type='modified')
        torch.cuda.synchronize()
        del ws
        assert torch.equal(costs, c2) and torch.equal(grads, g2), storage
        c_ref, g_ref = mr.dense_loss(a.double().cpu().numpy(), labels, tl, ul, delay_penalty=LAM)
        if storage == torch.float32:
            assert not close(costs.cpu().numpy(), grads.cpu().numpy(), c_ref, g_ref, tl, ul, LAM)
    print("groups ok")


if __name__ == "__main__":
    {"hooks": hooks, "groups": groups}[sys.argv[1]]()
