"""Wide channel plans (channels_interval 40 .. 64, a multiple of 8) on the tensor cores, without a GPU: the planner's choices
through the host-only wunet_debug_plan_prec, the plans of the narrow widths unchanged field for field, the refusals outside the
supported range, and the ptxas report of the unit that holds the wide plans' own kernels (wunet_tc_wide.cu)."""
import json
import os
import re
import subprocess
import sys

import pytest

from wave_u_net_for_speech_enhancement_b200 import _lib, build

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
import gen_narrow_plans_golden as narrow  # noqa: E402

SMS = 132
SMEM_SM = 228 * 1024
BATCHES = [1, 2, 3, 17, 64, 128, 256, 1000]
TC_PRECISIONS = ["bf16", "fp16", "fp32_tc"]


def test_narrow_plans_are_unchanged(golden_dir):
    """Every plan test_plan_invariants covers (ci <= 32) is what the library chose before wide plans existed, refusals included."""
    with open(os.path.join(golden_dir, "plans_narrow.json")) as f:
        want = json.load(f)
    assert want["fields"] == _lib.PLAN_FIELDS and want["num_sms"] == SMS
    got = narrow.digests(narrow.record(_lib))
    assert got.keys() == want["groups"].keys()
    assert sum(g["plans"] for g in got.values()) == 6624
    bad = [g for g in want["groups"] if got[g] != want["groups"][g]]
    assert not bad, f"plans of (n, ci, precision) {bad} moved; tools/gen_narrow_plans_golden.py --dump lists them for a diff"


def chunks(c):
    return -(-c // 64)


def check_plan(n, ci, B, T, i, prec, d):
    ctx = (n, ci, B, T, i, prec, d)
    ks = 15 if i <= n else 5
    cout_ref = (i + 1) * ci if i < n else (n * ci if i == n else (2 * n - i + 1) * ci)
    assert d["Cout"] == cout_ref, ctx                    # no row-pair form (it would double Cout of block 1)
    if d["small"] == 2:
        assert prec != "fp32_tc" and d["L"] <= 16 and i != 2 * n, ctx
        N = d["L"] * d["Cout"]
        assert d["Nh"] % 16 == 0 and N % d["Nh"] == 0 and d["nsplit"] == N // d["Nh"], ctx
        assert d["m_tiles"] * 128 >= B and d["Nh"] <= 128, ctx
        assert 2 <= d["na"] <= 8 and d["na"] * (d["a_stage_bytes"] + d["b_stage_bytes"]) <= d["smem"] <= 227 * 1024, ctx
        return
    # every 64-channel chunk of both K segments has its own K-loop slot: no merged tail chunk (three positions per chunk in
    # split precision)
    assert d["nchunks"] == (3 if prec == "fp32_tc" else 1) * (chunks(d["Cin0"]) + chunks(d["Cin1"])), ctx
    assert d["Nh"] % 16 == 0 and 16 <= d["Nh"] <= (64 if d["small"] else 128), ctx
    assert (d["nsplit"] - 1) * d["Nh"] < d["Npad"] <= d["nsplit"] * d["Nh"], ctx
    assert d["Nstride"] >= d["Nh"] and d["Nstride"] % 32 == 0, ctx
    assert d["MT"] == 1 and d["nacc"] == 1 and d["per_sm"] <= (2 if d["small"] else 1), ctx
    assert d["smem"] <= 227 * 1024 and d["per_sm"] * (d["smem"] + 1024) <= SMEM_SM, ctx
    assert d["na"] * d["a_stage_bytes"] + d["nb"] * d["b_stage_bytes"] <= d["smem"], ctx
    assert 2 <= d["na"] <= 4 or (d["na"] == 1 and d["small"] == 0), ctx
    assert d["a_tx_bytes"] <= d["a_stage_bytes"] and d["rows_used"] * 128 <= d["a_stage_bytes"], ctx
    assert d["a_stage_bytes"] % 1024 == 0 and d["b_stage_bytes"] % 1024 == 0, ctx
    assert 1 <= d["tg"] <= ks and d["tg"] * d["ngroups"] >= ks, ctx
    assert d["b_stage_bytes"] >= d["Nh"] * 128 * d["tg"], ctx
    if d["resident"]:
        assert d["nb"] == d["nchunks"] * d["ngroups"] and d["ngroups"] == 1, ctx
    else:
        assert 2 <= d["nb"] <= 8, ctx
    if d["packed"]:
        assert d["L"] < 128 and d["S"] == d["L"] + ks - 1, ctx
        assert 1 <= d["FR"] <= B and d["m_tiles"] * d["FR"] >= B, ctx
        assert (d["FR"] - 1) * d["S"] + d["L"] <= 128 * d["MT"], ctx
    else:
        assert d["tiles_per_frame"] * 128 * d["MT"] >= d["L"], ctx
        assert (d["tiles_per_frame"] - 1) * 128 * d["MT"] < d["L"], ctx
        assert d["m_tiles"] == B * d["tiles_per_frame"], ctx
    tiles = d["m_tiles"] * d["nsplit"]
    assert 1 <= d["grid"] <= min(tiles, SMS * d["per_sm"]), ctx
    assert d["threads"] * d["per_sm"] <= 2048 and d["threads"] % 32 == 0, ctx
    if i == 2 * n:                                      # fused head: the whole channel range of full frames in one CTA
        assert d["nsplit"] == 1 and not d["packed"] and d["Cout"] <= 64, ctx


@pytest.mark.parametrize("ci", [40, 48, 56, 64])
@pytest.mark.parametrize("n", [4, 8, 12])
@pytest.mark.parametrize("B", BATCHES)
def test_wide_plan_invariants(n, ci, B, monkeypatch):
    for k in ("WUNET_TC_OVR", "WUNET_TC_PAIR", "WUNET_TC_MERGE", "WUNET_TC_GEMM", "WUNET_TC_ENC0"):
        monkeypatch.delenv(k, raising=False)
    for T in narrow.lengths(n):
        for prec in TC_PRECISIONS:
            if T < 128:
                with pytest.raises(_lib.WunetError, match="at least 128 samples"):
                    _lib.debug_plan(n, ci, B, T, 2 * n, SMS, precision=prec)
                continue
            for i in range(1, 2 * n + 1):
                d = _lib.debug_plan(n, ci, B, T, i, SMS, precision=prec)
                check_plan(n, ci, B, T, i, prec, d)
                if prec == "fp16":                      # fp16 runs the bf16 plan
                    assert d == _lib.debug_plan(n, ci, B, T, i, SMS, precision="bf16")


def test_narrow_forms_are_off_for_wide_plans(monkeypatch):
    """The row-pair block 1, the merged decoder tail and the group-of-8 block 0 stay narrow-only, even where asked for."""
    monkeypatch.setenv("WUNET_TC_PAIR", "3")
    monkeypatch.setenv("WUNET_TC_MERGE", "1")
    for ci in (40, 48, 56, 64):
        d = _lib.debug_plan(12, ci, 256, 16384, 1, SMS)
        assert (d["L"], d["Cin0"], d["Cout"]) == (8192, ci, 2 * ci)          # the plain 15-tap block
        # ci = 40: the last block's tails (80 % 64 = 16 upsampled + 40 skip channels) would fit one merged chunk at a narrow width
        d = _lib.debug_plan(12, ci, 256, 16384, 24, SMS)
        assert d["nchunks"] == chunks(2 * ci) + chunks(ci), d
    monkeypatch.setenv("WUNET_TC_ENC0", "1")
    with pytest.raises(_lib.WunetError, match="group-of-8"):
        _lib.debug_plan(12, 40, 256, 16384, 0, SMS)
    assert _lib.debug_plan(12, 24, 256, 16384, 0, SMS)["Cout"] == 192       # still offered at 24


def test_split_precision_chunk_form():
    """The middle decoders of 12 layers at ci >= 48 have more than 48 split-precision positions (3 per 64-channel chunk): they
    are planned in the chunk form, up to 144 positions; narrower blocks keep the position form."""
    d = _lib.debug_plan(12, 48, 256, 16384, 13, SMS, precision="fp32_tc")
    assert (d["Cin0"], d["Cin1"], d["nchunks"]) == (576, 576, 54)
    d = _lib.debug_plan(12, 64, 256, 16384, 13, SMS, precision="fp32_tc")
    assert (d["Cin0"], d["Cin1"], d["nchunks"]) == (768, 768, 72)
    assert _lib.debug_plan(12, 40, 256, 16384, 13, SMS, precision="fp32_tc")["nchunks"] == 48


@pytest.mark.parametrize("prec", TC_PRECISIONS)
def test_outside_the_range_is_refused(prec):
    with pytest.raises(_lib.WunetError, match="<= 64"):
        _lib.debug_plan(12, 72, 256, 16384, 3, SMS, precision=prec)
    with pytest.raises(_lib.WunetError, match="% 8 == 0"):
        _lib.debug_plan(12, 44, 256, 16384, 3, SMS, precision=prec)


def _nvcc():
    try:
        return build.nvcc_path()
    except RuntimeError:
        return None


@pytest.mark.skipif(_nvcc() is None, reason="needs nvcc")
def test_wide_unit_compiles_without_spills_or_wgmma_serialisation(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DWUNET_BUILD", "-Xptxas", "-v", "-c",
           os.path.join(build.CSRC, "wunet_tc_wide.cu"), "-o", str(tmp_path / "wunet_tc_wide.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = r.stdout + r.stderr
    assert r.returncode == 0, log[-4000:]
    entries = re.findall(r"Compiling entry function '(\w+)'", log)
    assert len(entries) == 6 and sum("enc0_wide_kernel" in e for e in entries) == 3, entries
    assert sum("conv_tc_kernel" in e for e in entries) == 2 and any("pack_tc_split_wide_kernel" in e for e in entries), entries
    bad = [line for line in log.splitlines() if re.search(r"C75(19|20)", line)]
    assert not bad, "\n".join(bad[:10])
    assert not re.search(r"[1-9]\d* bytes spill stores", log), log[-4000:]
