"""The fp32 residual epilogues of the 128 x 256 GEMM kernel compile without local-memory spills (ptxas -v of
gemm_wide_resid.cu under the library's flags)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pigeon_b200", "csrc")


def test_wide_residual_kernels_do_not_spill(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    from pigeon_b200 import _build
    assert "gemm_wide_resid.cu" in _build.SOURCES
    r = subprocess.run([nvcc, *_build._flags(), "-Xptxas", "-v", "-I", os.path.join(ROOT, "include"), "-c",
                        os.path.join(CSRC, "gemm_wide_resid.cu"), "-o", str(tmp_path / "gemm_wide_resid.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    kernels = re.findall(r"Compiling entry function '(\S*gemm_wide_kernel\S*)'", r.stderr)
    assert len(kernels) == 4, kernels             # EPI_F32_BIAS_RESID, EPI_F32_BIAS_RESID_STATS x {fp16, bf16}
    reports = [l for l in r.stderr.splitlines() if "spill stores" in l]
    assert len(reports) >= 4
    assert all(re.search(r"\b0 bytes spill stores, 0 bytes spill loads", l) for l in reports), reports
