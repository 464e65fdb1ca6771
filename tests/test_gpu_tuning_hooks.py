"""Every kernel a tuning hook (RNNT_B200_* environment variables, README) selects, against the fp64 oracle.

A hook is read once per process, so each setting runs tests/hook_cases.py in a child process of its own.  Each case
asserts the child's verdicts, and that the hook changed the dispatch: a kernel only the hook launches appears in
the child's profiler trace, or the launch count / host-side policy shows the forced value.  Hooks that only
re-map work (batch groups, PDL, the factor ring depth, the chunk CTA size and lane mapping) must also give the
outputs of the default dispatch bit for bit; the others may change the rounding and are checked against the
oracle only.
"""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
TIMEOUT = 600

# name: (suite, environment, kernels that must appear, kernels that must not, outputs bitwise equal to the default)
CASES = {
    # additive joint
    "JOINT_SIMT_1": ("joint", {"RNNT_B200_JOINT_SIMT": "1"},
                     [r"joint_thin_kernel", r"joint_gemm_kernel<b200rnnt::EpiPartial, 32, 32>",
                      r"joint_gemm_kernel<b200rnnt::EpiPartial, 64, 32>", r"joint_gemm_kernel<b200rnnt::EpiGrad"],
                     [r"wg::gemm_kernel", r"grad_fused_kernel"], False),
    "JOINT_FUSED_0": ("joint", {"RNNT_B200_JOINT_FUSED": "0"},
                      [r"wg::gemm_kernel<3, 1, 64, 24>", r"wg::gemm_kernel<0, 1, 32, 24>"], [r"grad_fused_kernel"], False),
    "JOINT_SLICES_1": ("joint", {"RNNT_B200_JOINT_SLICES": "1"}, [], [], False),
    "JOINT_SLICES_7": ("joint", {"RNNT_B200_JOINT_SLICES": "7"}, [], [], False),
    "JOINT_SLICES_16": ("joint", {"RNNT_B200_JOINT_SLICES": "16"}, [], [], False),
    "DF_TILE_128": ("joint", {"RNNT_B200_DF_TILE": "128"}, [r"wg::gemm_kernel<3, 1, 128, 24>"], [], False),
    # smoothed additive joint (DESIGN.md §9): each hook must run the SMOOTH instantiation of its kernels
    "SMOOTHED_JOINT_SIMT_1": ("smoothed", {"RNNT_B200_JOINT_SIMT": "1"},
                              [r"joint_thin_kernel<true>", r"EpiGrad<true>", r"joint_stats_kernel<true>",
                               r"joint_gemm_kernel<b200rnnt::EpiPartial, 64, 32>"],
                              [r"wg::gemm_kernel", r"grad_fused_kernel"], False),
    "SMOOTHED_JOINT_FUSED_0": ("smoothed", {"RNNT_B200_JOINT_FUSED": "0"},
                               [r"wg::gemm_kernel<3, 1, 64, 24, b200rnnt::wg::Smooth>",
                                r"wg::gemm_kernel<0, 1, 32, 24, b200rnnt::wg::Smooth>", r"joint_stats_kernel<true>"],
                               [r"grad_fused_kernel"], False),
    "SMOOTHED_JOINT_SLICES_1": ("smoothed", {"RNNT_B200_JOINT_SLICES": "1"},
                                [r"grad_fused_kernel<32, 32, 3, true>", r"joint_stats_kernel<true>"], [], False),
    "SMOOTHED_JOINT_SLICES_7": ("smoothed", {"RNNT_B200_JOINT_SLICES": "7"},
                                [r"grad_fused_kernel<32, 32, 3, true>", r"joint_stats_kernel<true>"], [], False),
    "SMOOTHED_JOINT_SLICES_16": ("smoothed", {"RNNT_B200_JOINT_SLICES": "16"},
                                 [r"grad_fused_kernel<32, 32, 3, true>", r"joint_stats_kernel<true>"], [], False),
    "SMOOTHED_DF_TILE_128": ("smoothed", {"RNNT_B200_DF_TILE": "128"},
                             [r"wg::gemm_kernel<3, 1, 128, 24, b200rnnt::wg::Smooth>", r"joint_stats_kernel<true>"],
                             [], False),
    # dense loss
    "CHUNK_0": ("dense", {"RNNT_B200_CHUNK": "0"}, [r"grad_tile_kernel<float, 4, 2,", r"grad_tile_kernel<float, 2, 4,"],
                [r"grad_chunk_kernel", r"rowstats_chunk_kernel"], False),
    "CHUNK_NT_64": ("dense", {"RNNT_B200_CHUNK_NT": "64"}, [r"grad_chunk_kernel<float, 2, 64,"],
                    [r"grad_chunk_kernel<float, 2, 256,"], True),
    "CHUNK_NT_128": ("dense", {"RNNT_B200_CHUNK_NT": "128"}, [r"grad_chunk_kernel<float, 2, 128,"],
                     [r"grad_chunk_kernel<float, 2, 256,"], True),
    "CHUNK_TPR_1": ("dense", {"RNNT_B200_CHUNK_TPR": "1"}, [r"grad_chunk_kernel<float, 1, 256,"],
                    [r"grad_chunk_kernel<float, 2, 256,"], False),
    "CHUNK_TPR_4": ("dense", {"RNNT_B200_CHUNK_TPR": "4"}, [r"grad_chunk_kernel<float, 4, 256,"],
                    [r"grad_chunk_kernel<float, 2, 256,"], False),
    "CHUNK_TPR_8": ("dense", {"RNNT_B200_CHUNK_TPR": "8"}, [r"grad_chunk_kernel<float, 8, 256,"],
                    [r"grad_chunk_kernel<float, 2, 256,"], False),
    # fewer lanes than the default stage more rows per chunk: 51.2 KB of shared memory at V = 100 (and at V = 50
    # with one lane per row above), past the 48 KB a launch gets without opting in - the launch used to fail
    "CHUNK_TPR_2_chunk_over_48KB_shared": ("dense", {"RNNT_B200_CHUNK_TPR": "2"}, [r"grad_chunk_kernel<float, 2, 256,"],
                                           [r"grad_chunk_kernel<float, 4, 256,"], False),
    "CHUNK_MAP_0": ("dense", {"RNNT_B200_CHUNK_MAP": "0"}, [], [], True),
    "CHUNK_MAP_1": ("dense", {"RNNT_B200_CHUNK_MAP": "1"}, [], [], True),
    "LPR_32": ("dense", {"RNNT_B200_LPR": "32"}, [r"grad_tile_kernel<float, 4, 32,"], [r"grad_tile_kernel<float, 4, 16,"],
               False),
    "LAT_RING_16": ("dense", {"RNNT_B200_LAT_RING": "16"}, [r"lattice_lin_kernel<1, true, 16>"],
                    [r"lattice_lin_kernel<1, true, 8>"], True),
    "LAT_RING_32": ("dense", {"RNNT_B200_LAT_RING": "32"}, [r"lattice_lin_kernel<1, true, 32>"],
                    [r"lattice_lin_kernel<1, true, 8>"], True),
    "GROUPS_2": ("dense", {"RNNT_B200_GROUPS": "2"}, [], [], True),
    "GROUPS_3": ("dense", {"RNNT_B200_GROUPS": "3"}, [], [], True),
    "GROUPS_8": ("dense", {"RNNT_B200_GROUPS": "8"}, [], [], True),
    "PDL_1": ("dense", {"RNNT_B200_PDL": "1"}, [], [], True),
    # pruned loss (DESIGN.md §8): each hook must run the PRUNED instantiation (last template argument true) it selects
    "PRUNED_CHUNK_0": ("pruned", {"RNNT_B200_CHUNK": "0"},
                       [r"rowstats_tile_kernel<float, 4, 2, float, true>",
                        r"grad_tile_kernel<float, 4, 2, false, float, false, true>",
                        r"grad_tile_kernel<float, 2, 4, false, float, false, true>",
                        r"grad_tile_kernel<float, 4, 4, false, float, false, true>"],
                       [r"grad_chunk_kernel", r"rowstats_chunk_kernel"], False),
    "PRUNED_CHUNK_NT_64": ("pruned", {"RNNT_B200_CHUNK_NT": "64"},
                           [r"rowstats_chunk_kernel<float, 2, 64, true>",
                            r"grad_chunk_kernel<float, 2, 64, false, false, true>"],
                           [r"grad_chunk_kernel<float, 2, 256,"], True),
    "PRUNED_CHUNK_NT_128": ("pruned", {"RNNT_B200_CHUNK_NT": "128"},
                            [r"rowstats_chunk_kernel<float, 2, 128, true>",
                             r"grad_chunk_kernel<float, 2, 128, false, false, true>"],
                            [r"grad_chunk_kernel<float, 2, 256,"], True),
    "PRUNED_CHUNK_TPR_1": ("pruned", {"RNNT_B200_CHUNK_TPR": "1"},
                           [r"rowstats_chunk_kernel<float, 1, 256, true>",
                            r"grad_chunk_kernel<float, 1, 256, false, false, true>"],
                           [r"grad_chunk_kernel<float, 2, 256,"], False),
    "PRUNED_CHUNK_TPR_2": ("pruned", {"RNNT_B200_CHUNK_TPR": "2"},
                           [r"grad_chunk_kernel<float, 2, 256, false, false, true>"],
                           [r"grad_chunk_kernel<float, 4, 256,"], False),
    "PRUNED_CHUNK_TPR_4": ("pruned", {"RNNT_B200_CHUNK_TPR": "4"},
                           [r"rowstats_chunk_kernel<float, 4, 256, true>",
                            r"grad_chunk_kernel<float, 4, 256, false, false, true>"],
                           [r"grad_chunk_kernel<float, 2, 256,"], False),
    "PRUNED_CHUNK_TPR_8": ("pruned", {"RNNT_B200_CHUNK_TPR": "8"},
                           [r"rowstats_chunk_kernel<float, 8, 256, true>",
                            r"grad_chunk_kernel<float, 8, 256, false, false, true>"],
                           [r"grad_chunk_kernel<float, 2, 256,"], False),
    "PRUNED_CHUNK_MAP_0": ("pruned", {"RNNT_B200_CHUNK_MAP": "0"},
                           [r"grad_chunk_kernel<float, 2, 256, false, false, true>"], [], True),
    "PRUNED_CHUNK_MAP_1": ("pruned", {"RNNT_B200_CHUNK_MAP": "1"},
                           [r"grad_chunk_kernel<float, 2, 256, false, false, true>"], [], True),
    "PRUNED_LPR_32": ("pruned", {"RNNT_B200_LPR": "32"},
                      [r"rowstats_tile_kernel<float, 4, 32, float, true>",
                       r"grad_tile_kernel<float, 4, 32, false, float, false, true>"],
                      [r"grad_tile_kernel<float, 4, 16,"], False),
    "PRUNED_LAT_RING_16": ("pruned", {"RNNT_B200_LAT_RING": "16"},
                           [r"lattice_lin_kernel<1, true, 16>",
                            r"grad_chunk_kernel<float, 2, 256, false, false, true>"],
                           [r"lattice_lin_kernel<1, true, 8>"], True),
    "PRUNED_LAT_RING_32": ("pruned", {"RNNT_B200_LAT_RING": "32"},
                           [r"lattice_lin_kernel<1, true, 32>",
                            r"grad_chunk_kernel<float, 2, 256, false, false, true>"],
                           [r"lattice_lin_kernel<1, true, 8>"], True),
    "PRUNED_GROUPS_2": ("pruned", {"RNNT_B200_GROUPS": "2"},
                        [r"grad_chunk_kernel<float, 2, 256, false, false, true>"], [], True),
    "PRUNED_GROUPS_3": ("pruned", {"RNNT_B200_GROUPS": "3"},
                        [r"grad_chunk_kernel<float, 2, 256, false, false, true>"], [], True),
    "PRUNED_GROUPS_8": ("pruned", {"RNNT_B200_GROUPS": "8"},
                        [r"grad_chunk_kernel<float, 2, 256, false, false, true>"], [], True),
    "PRUNED_PDL_1": ("pruned", {"RNNT_B200_PDL": "1"},
                     [r"grad_chunk_kernel<float, 2, 256, false, false, true>"], [], True),
}
STREAMING = ("rowstats_chunk_kernel", "rowstats_tile_kernel", "rowstats_row_kernel", "grad_chunk_kernel",
             "grad_tile_kernel", "grad_row_kernel")


def norm(name):
    """One spelling of template arguments whichever demangler produced the name: 2 / true, not (int)2 / (bool)1."""
    name = re.sub(r"\((?:int|unsigned int)\)(-?\d+)", r"\1", name)
    return name.replace("(bool)0", "false").replace("(bool)1", "true")


def run_child(suite, env_extra, out_dir):
    env = {k: v for k, v in os.environ.items() if not k.startswith("RNNT_B200_")}
    env.update(env_extra)
    os.makedirs(out_dir, exist_ok=True)
    r = subprocess.run([sys.executable, os.path.join(HERE, "hook_cases.py"), suite, out_dir], env=env,
                       capture_output=True, text=True, timeout=TIMEOUT)
    assert r.returncode == 0, "hook child failed (%s):\n%s\n%s" % (env_extra, r.stdout[-4000:], r.stderr[-4000:])
    rep = json.loads(r.stdout.strip().splitlines()[-1])
    rep["kernels"] = [norm(k) for k in rep["kernels"]]
    return rep


@pytest.fixture(scope="module")
def baseline(tmp_path_factory):
    """The default dispatch, one child per suite (no hook set)."""
    out = {}
    for suite in ("dense", "joint", "smoothed", "pruned"):
        d = str(tmp_path_factory.mktemp("baseline_" + suite))
        out[suite] = (run_child(suite, {}, d), d)
    return out


def test_default_dispatch_matches_the_oracle(baseline):
    for suite, (rep, _) in baseline.items():
        for name, res in rep["shapes"].items():
            assert res["ok"], (suite, name, res["problems"])
    dense = baseline["dense"][0]
    assert dense["policy"]["pdl"] == 0
    assert all(res["launches"] == 3 for res in dense["shapes"].values())
    assert any("grad_fused_kernel" in k for k in baseline["joint"][0]["kernels"])
    assert any("grad_fused_kernel<32, 32, 3, true>" in k for k in baseline["smoothed"][0]["kernels"])
    pruned = baseline["pruned"][0]
    assert all(res["launches"] == 4 for res in pruned["shapes"].values())   # the log-zero fill, then the three
    streaming = [k.split("(")[0] for k in pruned["kernels"] if any(f in k for f in STREAMING)]
    assert len(streaming) == 6 and all(k.endswith(", true>") for k in streaming), streaming


@pytest.mark.parametrize("case", list(CASES))
def test_hook(case, baseline, tmp_path):
    suite, env, present, absent, bitwise = CASES[case]
    rep = run_child(suite, env, str(tmp_path))
    for name, res in rep["shapes"].items():
        assert res["ok"], (case, name, res["problems"])
    kernels = rep["kernels"]
    for pat in present:
        assert any(pat in k for k in kernels), (case, pat, [k for k in kernels if "b200rnnt" in k])
    for pat in absent:
        assert not any(pat in k for k in kernels), (case, pat)
    base_rep, base_dir = baseline[suite]
    pol, base_pol = rep["policy"], base_rep["policy"]
    # hooks that leave the kernel names alone: the launch count or the host-side policy shows the forced value
    key, value = next(iter(env.items()))
    if key == "RNNT_B200_JOINT_SLICES":
        assert all(pol[k] == int(value) for k in pol if k.startswith("slices_"))
        assert any(base_pol[k] != int(value) for k in base_pol if k.startswith("slices_"))
    elif key == "RNNT_B200_CHUNK_MAP":
        maps = [k for k in pol if k.startswith("map_V") and base_pol["default_" + k] != pol[k]]
        assert all(pol[k] == int(value) for k in pol if k.startswith("map_V"))
        assert maps, "no shape whose default mapping differs from the forced one"
    elif key == "RNNT_B200_GROUPS":
        fill = 1 if suite == "pruned" else 0   # a pruned call fills the whole lattice once, before every group
        assert all(res["launches"] == fill + 3 * int(value) for res in rep["shapes"].values()), rep["shapes"]
    elif key == "RNNT_B200_PDL":
        assert pol["pdl"] == 1
    elif key == "RNNT_B200_LAT_RING":
        assert pol["ring_U301"] == int(value) and base_pol["ring_U301"] == 8
    if bitwise:
        for name in rep["shapes"]:
            a, b = np.load(os.path.join(str(tmp_path), name + ".npz")), np.load(os.path.join(base_dir, name + ".npz"))
            for k in a.files:
                assert np.array_equal(a[k], b[k]), (case, name, k)
