"""CPU tests of the error / Jacobian export's host side: argument checks that need no device, the refusal without a CUDA
device (no CPU fallback), and the façade's new methods compiling and linking in both flavours."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from pop_up_slam_b200 import capi, graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


def test_host_checks_need_no_device():
    a = GpuGraphAPI()
    with pytest.raises(capi.ApiError, match="no live factors"):
        a.weighted_errors()
    g = gg.make_config(1, seed=0)
    ids = gg.build_bulk(a, g)
    rows, cols = a.jacobian_dims()
    assert (rows, cols) == (g.dims()["rows"], g.dims()["state_dim"])
    a.remove_factor(int(ids["pp_fids"][0]))
    assert a.jacobian_dims() == (rows - 3, cols)
    with pytest.raises(capi.ApiError, match="bad factor id"):
        a.factor_errors([int(ids["pp_fids"][0])])


@pytest.mark.skipif(not no_gpu(), reason="a CUDA device is present")
def test_export_entry_points_refuse_without_a_gpu():
    g = gg.make_config(1, seed=0)
    a = GpuGraphAPI()
    ids = gg.build_bulk(a, g)
    for call in (a.weighted_errors, a.jacobian, a.normalized_chi2, lambda: a.local_chi2(3),
                 lambda: a.factor_errors(ids["pp_fids"][:2])):
        with pytest.raises(capi.ApiError, match="no CUDA device"):
            call()


@pytest.mark.skipif(shutil.which("g++") is None, reason="no host C++ compiler")
@pytest.mark.parametrize("eigen", [False, True])
def test_facade_export_methods_compile_and_link(tmp_path, eigen):
    src = os.path.join(ROOT, "tests", "facade_export_replay.cpp")
    out = tmp_path / ("replay_eigen" if eigen else "replay")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), src, "-o", str(out),
           "-L", os.path.join(ROOT, "pop_up_slam_b200"), "-lpopup_gpu", "-Wl,-rpath," + os.path.join(ROOT, "pop_up_slam_b200")]
    if eigen:
        cmd[1:1] = ["-DISAM_FACADE_USE_EIGEN", "-I", os.path.join(ROOT, "oracle", "ref_shim")]
    subprocess.check_call(cmd)
    if no_gpu():   # the replay runs to the first device call and reports the refusal
        r = subprocess.run([str(out)], capture_output=True, text=True)
        assert r.returncode != 0 and "no CUDA device" in (r.stdout + r.stderr)
