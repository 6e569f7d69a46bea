"""The tensor-core kernels issue their wgmma instructions back to back. When a branch that ptxas cannot prove warpgroup-uniform
sits among them, ptxas waits for each MMA before issuing the next (C7520) or guards the accumulator registers with extra
warpgroup arrives (C7519), and the tensor cores run one instruction at a time. The guard compiles wunet_tc.cu for sm_90a with
ptxas in verbose mode (into a temporary directory, so the in-tree library is untouched) and rejects either diagnostic. No GPU
needed; skipped when nvcc is missing."""
import os
import re
import subprocess

import pytest

from wave_u_net_for_speech_enhancement_b200 import build


def _nvcc():
    try:
        return build.nvcc_path()
    except RuntimeError:
        return None


@pytest.mark.skipif(_nvcc() is None, reason="needs nvcc")
def test_tc_kernels_do_not_serialise_wgmma(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DWUNET_BUILD", "-Xptxas", "-v",
           "-c", os.path.join(build.CSRC, "wunet_tc.cu"), "-o", str(tmp_path / "wunet_tc.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = r.stdout + r.stderr
    assert r.returncode == 0, log[-4000:]
    # the verbose report covers both kernels (the diagnostics below would otherwise pass vacuously)
    assert "conv_tc_kernel" in log and "gemm_tc_kernel" in log
    bad = [line for line in log.splitlines() if re.search(r"C75(19|20)", line)]
    assert not bad, "\n".join(bad[:10])
