"""CPU: the work decomposition of the decode kernels (tiles x K slices per warp, cluster-local sub-plans, attention item
plans) covers every element exactly once for every supported geometry.  The planning functions are `__host__ __device__`
in csrc/decode_common.cuh; a small host program built with nvcc exercises them (no GPU needed)."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="nvcc not available")
def test_decode_work_decomposition_covers_everything_once(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = tmp_path / "plan_check"
    src = os.path.join(ROOT, "tests", "dev", "plan_check.cu")
    build = subprocess.run([nvcc, "-std=c++17", "-O1", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a",
                            "-I", os.path.join(ROOT, "include"), "-o", str(exe), src], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stderr[-2000:]
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0 and run.stdout.strip().endswith("OK"), run.stdout[-2000:]
