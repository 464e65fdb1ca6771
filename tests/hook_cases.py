"""Child process of test_gpu_tuning_hooks.py: runs one suite of shapes through the library with the tuning hooks
(RNNT_B200_* environment variables, README) already set in its environment, and checks each against the fp64 oracle.

    python tests/hook_cases.py {dense|joint|smoothed|pruned} OUT_DIR

"smoothed" runs the JOINT shapes with lm_only_scale 0.25 and am_only_scale 0.1 (DESIGN.md §9) and checks them
against the closed-form fp64 reference (tests/smoothed_reference.py).  "pruned" runs the DENSE shapes as pruned
calls (DESIGN.md §8) with R = 3 rows per frame over windows from random_monotone_ranges, and checks them against
the fp64 reference (tests/pruned_reference.py).

A hook is read once per process into a static, so every hook setting needs a process of its own.  Saves each
shape's costs and gradients to OUT_DIR/<shape>.npz and prints one JSON line:
    {"suite", "shapes": {name: {"ok", "problems", "launches"}}, "kernels": [...], "policy": {...}}
"kernels" are the CUDA kernels the calls launched, from torch.profiler's CUDA activity trace; "policy" is what
rnnt_b200_debug_policy reports for the hooks that leave no other trace.
"""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "warp-transducer_b200"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import pruned_reference  # noqa: E402
import smoothed_reference  # noqa: E402
from joint_reference import grad_mismatch, reference as joint_reference  # noqa: E402
from oracle import pyoracle  # noqa: E402
from test_gpu_add_joint_smoothed import FLOOR_DENSE_AM  # noqa: E402

# (N, T, U, V): N = 10 >= 8 so that RNNT_B200_GROUPS applies (uneven groups for 3 and 8); full calls with gradients
DENSE = {
    "V28_chunk": (10, 12, 6, 28),        # chunk kernels, 2 lanes per row, lane-adjacent mapping by default
    "V50_chunk": (10, 10, 5, 50),        # chunk kernels, pairs, slice-major mapping by default
    "V100_chunk": (10, 6, 4, 100),       # chunk kernels, 4 lanes per row: 25.6 KB chunks, 51.2 KB at 2 lanes
    "V300_tile": (10, 7, 4, 300),        # register-tile kernels, 16 lanes per row by default
    "U301_multiwarp": (10, 6, 301, 50),  # multi-warp lattice wavefront (factor ring), grouped wavefronts
}
# (N, T, U, V): the four SIMT branches (V < / >= 512, U <= / > 32) and the tensor-core paths
JOINT = {
    "U20_V520": (2, 70, 20, 520),        # fused gradient (tensor cores) / joint_thin_kernel (SIMT)
    "U10_V100": (2, 30, 10, 100),        # fused, MODE 0 / joint_gemm_kernel 32-wide
    "U40_T80_V200": (2, 80, 40, 200),    # two-kernel gradient, dF over 80 frames (two 64-wide tiles or one 128)
    "U40_V1000": (2, 24, 40, 1000),      # two-kernel gradient, 3 split-K slabs / joint_thin_kernel
    "U8_V5121": (2, 16, 8, 5121),        # 16 split-K slabs, the last empty
}
SMOOTH = (0.25, 0.1)   # (lm_only_scale, am_only_scale) of the smoothed suite
# dG's dense-column floor of the smoothed suite (joint_reference's default, FLOOR_DENSE_AM for am_only_scale > 0), and
# per shape where a hook needs more.  U8_V5121: RNNT_B200_JOINT_SLICES=1 sums all 5121 columns of S in one
# tensor-core accumulation instead of 16 slabs; measured 1.79e-7 on an H100 80GB HBM3 at 700 W.
SMOOTH_FLOOR_DENSE = {"U8_V5121": 3e-7}
PRUNED_R = 3   # rows per frame of the pruned suite


def inputs(name, shape, joint, pruned=False):
    seed = sum(map(ord, name))
    rng = np.random.default_rng(seed)
    N, T, U, V = shape
    labels = rng.integers(1, V, size=(N, U - 1)).astype(np.int32)
    tl = rng.integers(max(1, T // 2), T + 1, size=N).astype(np.int32)
    ul = rng.integers(0, U, size=N).astype(np.int32)
    tl[0], ul[0] = T, U - 1
    if joint:
        x = ((rng.standard_normal((N, T, V)) * 2).astype(np.float32), (rng.standard_normal((N, U, V)) * 2).astype(np.float32))
    elif pruned:
        # utterance 0 keeps U_b = U, without a path where R - 1 labels per frame cannot reach it (U301: dead chains
        # across every warp of the wavefront); the others are cut to what their windows can reach
        ul[1:] = np.minimum(ul[1:], (tl[1:] - 1) * (PRUNED_R - 1))
        ranges = pruned_reference.random_monotone_ranges(rng, tl, ul, T, PRUNED_R)
        x = ((rng.standard_normal((N, T, PRUNED_R, V)) * 2).astype(np.float32), ranges)
    else:
        x = (rng.standard_normal((N, T, U, V)) * 2).astype(np.float32)
    return x, labels, tl, ul


def run_dense(wr, acts, labels, tl, ul):
    N = acts.shape[0]
    a = torch.tensor(acts, device="cuda")
    lab, tld, uld = (torch.as_tensor(x).cuda() for x in (labels, tl, ul))
    costs = torch.empty(N, device="cuda")
    grads = torch.full_like(a, float("nan"))
    ws = wr.gpu_rnnt_async(a, lab, tld, uld, costs, grads, 0)
    launches = wr.last_launch_count()
    torch.cuda.synchronize()
    del ws
    return costs.cpu().numpy(), grads.cpu().numpy(), launches


def run_pruned(wr, logits, ranges, labels, tl, ul, U):
    """The full pruned call (rnnt_b200_pruned_loss_async_ex) over the whole lattice width U."""
    from warprnnt_pytorch.pruned import pruned_workspace_size
    N, T, R, V = logits.shape
    x = torch.tensor(logits, device="cuda")
    rg, lab, tld, uld = (torch.as_tensor(a).cuda() for a in (ranges, labels, tl, ul))
    costs = torch.empty(N, device="cuda")
    grads = torch.full_like(x, float("nan"))
    ws = torch.empty(pruned_workspace_size(T, U, R, N, 4), dtype=torch.uint8, device="cuda")
    opt = wr.rnntOptions(loc=1, num_threads=0, stream=torch.cuda.current_stream().cuda_stream, blank_label=0,
                         maxT=T, maxU=U, batch_first=True)
    st = wr.lib().rnnt_b200_pruned_loss_async_ex(0, 0, x.data_ptr(), grads.data_ptr(), rg.data_ptr(), R,
                                                 lab.data_ptr(), uld.data_ptr(), tld.data_ptr(), V, N,
                                                 costs.data_ptr(), 1.0, wr.rnntGradOptions(0.0, 0.0), ws.data_ptr(),
                                                 opt)
    assert st == 0, wr.status_string(st)
    launches = wr.last_launch_count()
    torch.cuda.synchronize()
    del ws
    return costs.cpu().numpy(), grads.cpu().numpy(), launches


def check_pruned(out, x, labels, tl, ul):
    costs, grads = out
    c_ref, g_ref = pruned_reference.pruned_loss(x[0].astype(np.float64), labels, tl, ul, x[1], 0)
    problems = []
    fin = np.isfinite(c_ref)
    if not (np.array_equal(np.isfinite(costs), fin) and np.allclose(costs[fin], c_ref[fin], rtol=1e-5, atol=1e-5)):
        problems.append("costs: %s against %s" % (costs.tolist(), c_ref.tolist()))
    if np.isnan(grads).any() or not np.allclose(grads, g_ref, rtol=1e-4, atol=1e-6):
        problems.append("grads: max |err| %.3g" % np.nanmax(np.abs(grads - g_ref)))
    if grads[~fin].any():
        problems.append("an utterance without a path has a gradient")
    return problems


def run_joint(wr, trans, pred, labels, tl, ul):
    from warprnnt_pytorch.joint import add_joint_call
    N, T, V = trans.shape
    U = pred.shape[1]
    lab, tld, uld = (torch.as_tensor(x).cuda() for x in (labels, tl, ul))
    costs = torch.empty(N, device="cuda")
    dF = torch.full((N, T, V), float("nan"), device="cuda")
    dG = torch.full((N, U, V), float("nan"), device="cuda")
    ws = add_joint_call(torch.tensor(trans, device="cuda"), torch.tensor(pred, device="cuda"), lab, tld, uld, costs,
                        dF, dG, 0, 1.0)
    launches = wr.last_launch_count()
    torch.cuda.synchronize()
    del ws
    return costs.cpu().numpy(), dF.cpu().numpy(), dG.cpu().numpy(), launches


def run_smoothed(wr, trans, pred, labels, tl, ul):
    from warprnnt_pytorch.joint import add_joint_rnnt_loss
    tt = torch.tensor(trans, device="cuda", requires_grad=True)
    pp = torch.tensor(pred, device="cuda", requires_grad=True)
    lab, tld, uld = (torch.as_tensor(x).cuda() for x in (labels, tl, ul))
    out = add_joint_rnnt_loss(tt, pp, lab, tld, uld, 0, 'none', lm_only_scale=SMOOTH[0], am_only_scale=SMOOTH[1])
    out.sum().backward()
    launches = wr.last_launch_count()
    torch.cuda.synchronize()
    return out.detach().cpu().numpy(), tt.grad.cpu().numpy(), pp.grad.cpu().numpy(), launches


def check_smoothed(name, out, x, labels, tl, ul):
    costs, dF, dG = out
    c_ref, dF_ref, dG_ref = smoothed_reference.closed_form(x[0], x[1], labels, tl, ul, *SMOOTH)
    problems = []
    if not np.allclose(costs, c_ref, rtol=1e-5, atol=1e-5):
        problems.append("costs: max |err| %.3g" % np.abs(costs - c_ref).max())
    floor = SMOOTH_FLOOR_DENSE.get(name, FLOOR_DENSE_AM)
    problems += grad_mismatch(dF, dF_ref, tl, labels, ul, 0, "dF", floor_dense=floor)
    problems += grad_mismatch(dG, dG_ref, ul + 1, labels, ul, 0, "dG", floor_dense=floor)
    return problems


def check_dense(out, acts, labels, tl, ul):
    costs, grads = out
    c_ref, g_ref, _ = pyoracle.rnnt_logits(acts.astype(np.float64), labels, tl, ul, 0)
    problems = []
    if not np.allclose(costs, c_ref, rtol=1e-5, atol=1e-5):
        problems.append("costs: max |err| %.3g" % np.abs(costs - c_ref).max())
    if not np.allclose(grads, g_ref, rtol=1e-4, atol=1e-6):
        problems.append("grads: max |err| %.3g" % np.nanmax(np.abs(grads - g_ref)))
    return problems


def check_joint(out, x, labels, tl, ul):
    costs, dF, dG = out
    c_ref, dF_ref, dG_ref = joint_reference(x[0], x[1], labels, tl, ul, 0)
    problems = []
    if not np.allclose(costs, c_ref, rtol=1e-5, atol=1e-5):
        problems.append("costs: max |err| %.3g" % np.abs(costs - c_ref).max())
    problems += grad_mismatch(dF, dF_ref, tl, labels, ul, 0, "dF")
    problems += grad_mismatch(dG, dG_ref, ul + 1, labels, ul, 0, "dG")
    return problems


def main():
    suite, out_dir = sys.argv[1], sys.argv[2]
    import warprnnt_pytorch.warp_rnnt as wr
    lib = wr.lib()
    lib.rnnt_b200_debug_policy.restype = C.c_int
    lib.rnnt_b200_debug_policy.argtypes = [C.c_int, C.c_int, C.c_int]
    joint = suite in ("joint", "smoothed")
    pruned = suite == "pruned"
    if pruned:
        import warprnnt_pytorch.pruned  # noqa: F401  (argtypes of the pruned entries)
    shapes = JOINT if joint else DENSE
    run = {"dense": run_dense, "joint": run_joint, "smoothed": run_smoothed, "pruned": run_pruned}[suite]
    results, kernels = {}, set()
    for name, shape in shapes.items():
        x, labels, tl, ul = inputs(name, shape, joint, pruned)
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            if pruned:
                *out, launches = run(wr, *x, labels, tl, ul, shape[2])
            else:
                *out, launches = run(wr, *(x if joint else (x,)), labels, tl, ul)
        kernels.update(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
        if suite == "smoothed":
            problems = check_smoothed(name, out, x, labels, tl, ul)
        elif pruned:
            problems = check_pruned(out, x, labels, tl, ul)
        else:
            problems = (check_joint if joint else check_dense)(out, x, labels, tl, ul)
        keys = ("costs", "dF", "dG") if joint else ("costs", "grads")
        np.savez(os.path.join(out_dir, name + ".npz"), **dict(zip(keys, out)))
        results[name] = {"ok": not problems, "problems": problems, "launches": launches}
    policy = {"pdl": lib.rnnt_b200_debug_policy(7, 0, 0)}
    for name, (N, T, U, V) in shapes.items():
        policy["slices_V%d" % V] = lib.rnnt_b200_debug_policy(5, V, 0)
        if V * 4 <= 512:   # rows short enough for the chunk kernels
            policy["map_V%d" % V] = lib.rnnt_b200_debug_policy(6, V, 4)
            policy["default_map_V%d" % V] = lib.rnnt_b200_debug_policy(1, V, 4)
        policy["ring_U%d" % U] = lib.rnnt_b200_debug_policy(4, U, 0)
    print(json.dumps({"suite": suite, "shapes": results, "kernels": sorted(kernels), "policy": policy}))


if __name__ == "__main__":
    main()
