"""The 256-row form of the streamed-weight blocks (csrc/wunet_tc_m2.cu), without a GPU.

- The unit compiles for sm_90a with its wgmma issued back to back (no C7519 / C7520, see test_wgmma_issue_cpu.py), and each of its
  kernels keeps its two m64 accumulator blocks in registers: no spills, within the register budget ptxas gives the launch shape.
- The selection rule (wunet_debug_plan_m2) picks exactly the blocks that stream their weights and have enough 256-row units, and
  every geometry it picks fits in shared memory. The plan record itself (wunet_debug_plan) is covered by the plan goldens.
"""
import os
import re
import subprocess

import pytest

from wave_u_net_for_speech_enhancement_b200 import _lib, build

N, CI, B, T, SMS = 12, 24, 256, 16384, 132
# enc3, enc5, enc6, dec5, dec6, dec8 (enc4 and dec7 have 128 columns per CTA, more than the form's 96)
SELECTED = {3, 5, 6, 18, 19, 21}
SMEM_LIMIT = 227 * 1024


def _nvcc():
    try:
        return build.nvcc_path()
    except RuntimeError:
        return None


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in ("WUNET_TC_M2", "WUNET_TC_OVR", "WUNET_TC_GEMM", "WUNET_TC_PAIR", "WUNET_TC_ENC0", "WUNET_TC_MERGE"):
        monkeypatch.delenv(k, raising=False)


def m2(block, b=B, sms=SMS, precision="bf16", n=N, ci=CI, t=T):
    return _lib.debug_plan_m2(n, ci, b, t, block, sms, precision)


@pytest.mark.skipif(_nvcc() is None, reason="needs nvcc")
def test_m2_unit_compiles_without_serialised_wgmma_or_spills(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DWUNET_BUILD", "-Xptxas", "-v",
           "-c", os.path.join(build.CSRC, "wunet_tc_m2.cu"), "-o", str(tmp_path / "wunet_tc_m2.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = r.stdout + r.stderr
    assert r.returncode == 0, log[-4000:]
    bad = [line for line in log.splitlines() if re.search(r"C75(19|20)", line)]
    assert not bad, "\n".join(bad[:10])
    entries = re.findall(r"Compiling entry function '(\w+)'.*?\n(.*?spill stores.*?)\n.*?Used (\d+) registers", log, re.S)
    entries = [e for e in entries if "conv_tc_m2_kernel" in e[0]]
    # (bf16, fp16) x (encoder, decoder, decoder with a merged tail chunk)
    assert len(entries) == 6, log[-4000:]
    for name, spill, regs in entries:
        assert "0 bytes spill stores, 0 bytes spill loads" in spill, (name, spill)
        threads = 32 * (1 + 8 + (3 if "Lb1E" in name else 0))       # TMA warp, two consumer warpgroups, decoder producers
        # ptxas budgets whole warpgroups: 65536 registers over the threads rounded up to a multiple of 128
        assert int(regs) <= 65536 // (-(-threads // 128) * 128) // 8 * 8, (name, regs)


@pytest.mark.parametrize("precision", ("bf16", "fp16"))
def test_benchmark_shape_selects_the_streamed_blocks(precision):
    got = {i for i in range(1, 2 * N + 1) if m2(i, precision=precision)["selected"]}
    assert got == SELECTED
    for i in range(1, 2 * N + 1):
        p = _lib.debug_plan(N, CI, B, T, i, SMS, precision)
        d = m2(i, precision=precision)
        if i not in SELECTED:
            assert d == dict.fromkeys(_lib.M2_FIELDS, 0), (i, d)
            continue
        # a streamed, unpacked large-flavour block with whole 256-row units
        assert p["resident"] == 0 and p["packed"] == 0 and p["small"] == 0 and p["tiles_per_frame"] % 2 == 0, (i, p)
        assert d["units"] == B * p["tiles_per_frame"] // 2 * p["nsplit"] >= SMS, (i, d, p)
        assert d["grid"] == min(d["units"], SMS)
        assert d["smem"] <= SMEM_LIMIT, (i, d)
        assert d["na"] == p["na"] and 2 <= d["nb"] <= 8, (i, d)
        assert d["ngroups"] == -(-(15 if i <= N else 5) // d["tg"]), (i, d)


def test_the_benchmark_geometries():
    # enc3: 15 taps in three stages of five next to two 36 KB operand stages; the decoders at 96 columns: three 34 KB operand
    # stages and two stages of all five taps (227,328 bytes of ring)
    assert {k: m2(3)[k] for k in ("na", "nb", "tg")} == {"na": 2, "nb": 2, "tg": 5}
    for blk in (18, 21):
        assert {k: m2(blk)[k] for k in ("na", "nb", "tg")} == {"na": 3, "nb": 2, "tg": 5}


def test_small_batches_and_other_paths_select_nothing(monkeypatch):
    for i in range(1, 2 * N + 1):
        assert not m2(i, b=1)["selected"], i                        # latency_b1: the 128-row tiles keep every SM busy
        assert not m2(i, precision="fp32_tc")["selected"], i        # split precision keeps its forms
    monkeypatch.setenv("WUNET_TC_M2", "0")
    assert not any(m2(i)["selected"] for i in range(1, 2 * N + 1))


def test_a_streamed_override_on_a_resident_block_is_selected(monkeypatch):
    assert not m2(2)["selected"] and not m2(22)["selected"]
    monkeypatch.setenv("WUNET_TC_OVR", "2:res=0;22:res=0")
    for blk in (2, 22):
        assert _lib.debug_plan(N, CI, B, T, blk, SMS)["resident"] == 0
        d = m2(blk)
        assert d["selected"] and d["smem"] <= SMEM_LIMIT, (blk, d)


def test_every_selected_geometry_fits():
    for ci in (8, 16, 24, 32, 48, 64):
        for b in (1, 2, 3, 16, 64, 256):
            for i in range(1, 2 * N + 1):
                d = m2(i, b=b, ci=ci)
                if d["selected"]:
                    assert d["smem"] <= SMEM_LIMIT and d["nb"] >= 2 and d["units"] >= SMS, (ci, b, i, d)
