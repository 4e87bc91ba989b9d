"""The pass planner of fc_render3d_frames, fc_render3d_scene and fc_contour_build_slices (fidget_b200/csrc/cuda/
pass_plan.h) is plain host code: a host program compiled with nvcc replays scripted passes through it and prints the
ranges it takes, which must be the ones the overflow policy gives by hand."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

EXPECTED = {
    "a": "[0,1) [1,7) [7,10)",
    "b": "[0,1) [1,7) [1,4) [4,7) [7,10)",
    "c1": "[0,1) fail 1",             # error bit 0, one item: device_error gives FC_ERR_ARENA
    "c2": "[0,1) [1,9) fail 4",       # error bit 2 is no overflow: not split
    "d": "[0,3) [3,6) [6,9) [9,10)",
    "e": "[0,1) [1,3) [3,5) [5,7) [7,9) [9,10)",
    "f": "[0,1) [1,3) [3,5) [5,7) [7,9) [9,10)",
    "f_off": "[0,1) [1,9) [9,10)",
    "g": "[0,1) [1,7) [7,10)",        # an arena that grows after the planner is built sizes the later passes
}


@pytest.fixture(scope="module")
def passes(tmp_path_factory):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("pass_plan") / "pass_plan_check")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O1",
                    "-I", os.path.join(ROOT, "fidget_b200", "csrc", "cuda"), "-o", exe,
                    os.path.join(ROOT, "tests", "csrc", "pass_plan_check.cu")], check=True, capture_output=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.splitlines()
    return dict(line.split(" ", 1) for line in out)


@pytest.mark.parametrize("scenario", sorted(EXPECTED))
def test_pass_ranges(passes, scenario):
    assert passes[scenario] == EXPECTED[scenario]


def test_every_scenario_checked(passes):
    assert sorted(passes) == sorted(EXPECTED)
