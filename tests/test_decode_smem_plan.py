"""CPU: the shared-memory plan of the Llama-family decode launch (csrc/llama_decode_plan.cuh).  Llama-3-8B plans 16 sessions
per launch on 66 and 132 CTAs inside the sm_90 opt-in limit, with the reduction orders of the 8-session launch, and every
batch that had a plan before the third tier keeps it.  A small host program built with nvcc tabulates the plans (no GPU
needed)."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="nvcc not available")
def test_llama_decode_smem_plans(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = tmp_path / "decode_plan_check"
    src = os.path.join(ROOT, "tests", "dev", "decode_plan_check.cu")
    build = subprocess.run([nvcc, "-std=c++17", "-O1", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a",
                            "-I", os.path.join(ROOT, "include"), "-o", str(exe), src], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stderr[-2000:]
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0 and run.stdout.strip().endswith("OK"), run.stdout[-3000:]
    assert "llama-3-8b grid  66 B 16: kmax  4096 rg -1 kc 4096 slots 2 assoc_b  8 dynamic 224512 B" in run.stdout
