"""Each contraction of the additive joint against float64 on the fp32 operands it read on the GPU (tests/joint_stages.py):
J1 (Ef, Eg, mf, mg), S = Ef Eg^T with 1/S, and the dF / dG products with their blank and label terms, each within a
bound derived from the tf32 hi / lo split and the tensor core's fp32 accumulation, at the training shapes (long: the
two-kernel gradient over 151 label positions and 500 frames; C3: the fused gradient and 15 split-K slabs), the
two-kernel control shape, and vocabulary-tiled two-kernel shapes with MODE 3 and MODE 0 operands.

The workspace layout the reader assumes is checked against rnnt_b200_add_joint_workspace_size here without a GPU, and
on the GPU by every run (the reader asserts the size; J1 reads Ef / Eg / mf / mg at their offsets and must match).
"""
import json
import os
import subprocess
import sys

import pytest

import joint_stages as js

HERE = os.path.dirname(os.path.abspath(__file__))
STAGES = ("J1_f", "J1_g", "S", "dF", "dG")


def test_layout_ends_at_the_workspace_size():
    """carve_joint's sections as the reader lays them out end exactly where the C-ABI's workspace size does: fused
    (U <= 32: Wm padded to 32 label positions) and two-kernel widths, unaligned section sizes, the training shapes."""
    shapes = [(1, 1, 1, 1), (3, 7, 5, 11), (2, 33, 32, 129), (2, 10, 33, 64), (5, 17, 151, 501),
              (32, 500, 151, 500), (128, 150, 21, 5000), (1, 1000, 40, 64)] + list(js.SHAPES.values())
    for N, T, U, V in shapes:
        offsets, end = js.layout(N, T, U, V)
        assert end == js.workspace_size(N, T, U, V), (N, T, U, V)
        assert all(o % js.ALIGN == 0 for o in offsets.values())
        assert list(offsets) == sorted(offsets, key=offsets.get)


def check(name, ratios):
    bad = {k: ratios[k] for k in STAGES if not ratios[k] <= 1.0}
    if not ratios["inv_s_ulps"] <= 1:
        bad["inv_s_ulps"] = ratios["inv_s_ulps"]
    assert not bad, "%s: stages over their bound (|error| / bound): %s" % (name, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(js.SHAPES))
def test_stage_bounds(name):
    check(name, js.stage_ratios(*js.SHAPES[name]))


@pytest.mark.gpu
def test_stage_bounds_with_tuning_hooks():
    """The same shapes with 128-wide dF tiles and 3 split-K slabs of S (a hook is read once per process: a child)."""
    env = dict(os.environ, RNNT_B200_DF_TILE="128", RNNT_B200_JOINT_SLICES="3")
    r = subprocess.run([sys.executable, os.path.join(HERE, "joint_stages.py"), "--slices"] + list(js.SHAPES),
                       env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res.pop("slices") == {str(V): 3 for V in sorted({s[3] for s in js.SHAPES.values()})}
    for name in js.SHAPES:
        check(name + " (hooks)", res[name])
