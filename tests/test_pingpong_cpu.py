"""The ping-pong unit (csrc/wunet_tc_pp.cu) compiles for sm_90a with its wgmma issued back to back (no C7519 / C7520, see
test_wgmma_issue_cpu.py) and its kernels fit the launch bound of 416 threads at one CTA per SM without spilling: the two m64
accumulator blocks of a tile (2 x 40 fp32 registers per thread) stay in registers. No GPU needed; skipped without nvcc."""
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
def test_pingpong_unit_compiles_without_serialised_wgmma_or_spills(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DWUNET_BUILD", "-Xptxas", "-v",
           "-c", os.path.join(build.CSRC, "wunet_tc_pp.cu"), "-o", str(tmp_path / "wunet_tc_pp.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = r.stdout + r.stderr
    assert r.returncode == 0, log[-4000:]
    bad = [line for line in log.splitlines() if re.search(r"C75(19|20)", line)]
    assert not bad, "\n".join(bad[:10])
    # per kernel: the entry line, then its stack / spill line; four kernels (bf16, fp16) x (MG = 0, 1)
    entries = re.findall(r"Compiling entry function '(\w+)'.*?\n(.*?spill stores.*?)\n.*?Used (\d+) registers", log, re.S)
    entries = [e for e in entries if "conv_tc_pp_kernel" in e[0]]
    assert len(entries) == 4, log[-4000:]
    for name, spill, regs in entries:
        assert "0 bytes spill stores, 0 bytes spill loads" in spill, (name, spill)
        assert int(regs) <= 65536 // 416 // 8 * 8, (name, regs)
