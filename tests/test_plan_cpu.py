"""Host logic of the bf16 path: the per-block tiling decision (wunet_tc.cu: plan_block) queried through the C ABI's
host-only wunet_debug_plan — no GPU needed. Golden: the plan the library chooses on an H100 (132 SMs) for the benchmark
configuration; invariants: resource limits and coverage for a grid of shapes."""
import json
import os

import pytest

from wave_u_net_for_speech_enhancement_b200 import _lib

SMS = 132
SMEM_SM = 228 * 1024


def blocks(n):
    return range(1, 2 * n + 1)


def test_golden_plan_of_the_benchmark_config(golden_dir):
    g = json.load(open(os.path.join(golden_dir, "plan_n12_c24_b256.json")))
    name = {"res": "resident", "bulk": "bulk_store", "tmem": "tmem_cols"}
    for want in g["blocks"]:
        got = _lib.debug_plan(12, 24, 256, 16384, want["block"], g["num_sms"])
        for k, v in want.items():
            if k == "block":
                continue
            if k == "tiles":
                assert got["m_tiles"] * got["nsplit"] == v, (want["block"], k)
            else:
                assert got[name.get(k, k)] == v, (want["block"], k, got)


@pytest.mark.parametrize("n,ci", [(4, 8), (8, 16), (12, 24), (12, 32), (12, 8), (10, 24)])
@pytest.mark.parametrize("B", [1, 2, 3, 17, 64, 128, 256, 1000])
def test_plan_invariants(n, ci, B):
    for T in {1 << n, 4 << n, 16384 if 16384 % (1 << n) == 0 else 8 << n}:
        if T < 128:                             # the fused head works on full (unpacked) frames: rejected loudly
            with pytest.raises(_lib.WunetError, match="at least 128 samples"):
                _lib.debug_plan(n, ci, B, T, 2 * n, SMS)
            continue
        for i in blocks(n):
            d = _lib.debug_plan(n, ci, B, T, i, SMS)
            ks = 15 if i <= n else 5
            cout_ref = (i + 1) * ci if i < n else (n * ci if i == n else (2 * n - i + 1) * ci)
            pair = d["Cout"] == 2 * cout_ref            # row-pair mode (block 1 by default): half the rows, twice the columns,
            if pair:                                    # 9 taps for 15
                assert i == 1 and n >= 2 and d["L"] * 2 == T >> i and d["L"] >= 128, (n, ci, B, T, i, d)
                ks = 9
            else:
                assert d["Cout"] == cout_ref, (n, ci, B, T, i, d)
            ctx = (n, ci, B, T, i, d)
            if d["small"] == 2:
                # dense GEMM over frames (blocks of at most 16 samples): 128 frames x Nh columns per CTA, K = 64-channel chunks
                assert d["L"] <= 16 and i != 2 * n, ctx
                N = d["L"] * d["Cout"]
                assert d["Nh"] % 16 == 0 and N % d["Nh"] == 0 and d["nsplit"] == N // d["Nh"], ctx
                assert d["m_tiles"] * 128 >= B and d["Nh"] <= 128, ctx    # accumulators: registers of two consumer warpgroups
                assert 2 <= d["na"] <= 8 and d["na"] * (d["a_stage_bytes"] + d["b_stage_bytes"]) <= d["smem"] <= 227 * 1024, ctx
                cin = d["Cin0"] + d["Cin1"]
                assert d["nchunks"] >= -(-cin // 64), ctx
                continue
            # column tiling
            assert d["Nh"] % 16 == 0 and 16 <= d["Nh"] <= (64 if d["small"] else 128), ctx   # register accumulators
            assert (d["nsplit"] - 1) * d["Nh"] < d["Npad"] <= d["nsplit"] * d["Nh"], ctx
            assert d["Nstride"] >= d["Nh"] and d["Nstride"] % 32 == 0, ctx
            # one 128-row M tile per CTA, accumulators in the consumer warpgroups' registers
            assert d["MT"] == 1 and d["nacc"] == 1 and d["per_sm"] <= (2 if d["small"] else 1), ctx
            # shared memory: rings fit, every co-resident CTA (dynamic + 1 KB reserved) fits in the SM
            assert d["smem"] <= 227 * 1024, ctx
            assert d["per_sm"] * (d["smem"] + 1024) <= SMEM_SM, ctx
            assert d["na"] * d["a_stage_bytes"] + d["nb"] * d["b_stage_bytes"] <= d["smem"], ctx
            assert 2 <= d["na"] <= 4 or (d["na"] == 1 and d["small"] == 0), ctx
            assert d["a_tx_bytes"] <= d["a_stage_bytes"] and d["rows_used"] * 128 <= d["a_stage_bytes"], ctx
            assert d["a_stage_bytes"] % 1024 == 0 and d["b_stage_bytes"] % 1024 == 0, ctx
            # weight ring
            assert 1 <= d["tg"] <= ks and d["tg"] * d["ngroups"] >= ks, ctx
            assert d["b_stage_bytes"] >= d["Nh"] * 128 * d["tg"], ctx
            if d["resident"]:
                assert d["nb"] == d["nchunks"] * d["ngroups"] and d["ngroups"] == 1, ctx
            else:
                assert 2 <= d["nb"] <= 8, ctx
            # coverage of the output rows
            if d["packed"]:
                assert d["L"] < 128 and d["S"] == d["L"] + ks - 1, ctx
                assert 1 <= d["FR"] <= B and d["m_tiles"] * d["FR"] >= B, ctx
                assert (d["FR"] - 1) * d["S"] + d["L"] <= 128 * d["MT"], ctx
            else:
                assert d["tiles_per_frame"] * 128 * d["MT"] >= d["L"], ctx
                assert (d["tiles_per_frame"] - 1) * 128 * d["MT"] < d["L"], ctx
                assert d["m_tiles"] == B * d["tiles_per_frame"], ctx
            if d["bulk_store"]:
                assert not d["packed"] and d["nsplit"] == 1 and d["L"] % (128 * d["MT"]) == 0 and i != 2 * n, ctx
            # launch shape
            tiles = d["m_tiles"] * d["nsplit"]
            assert 1 <= d["grid"] <= min(tiles, SMS * d["per_sm"]), ctx
            assert d["threads"] * d["per_sm"] <= 2048 and d["threads"] % 32 == 0, ctx
            if i == 2 * n:                      # fused head: whole channel range of full frames in one CTA
                assert d["nsplit"] == 1 and not d["packed"] and d["Cout"] <= 32, ctx


def test_override_string(monkeypatch):
    base = _lib.debug_plan(12, 24, 256, 16384, 7, SMS)
    monkeypatch.setenv("WUNET_TC_OVR", "3:mt=1;7:small=1,nacc=1")
    d = _lib.debug_plan(12, 24, 256, 16384, 7, SMS)
    assert d["small"] == 1 and d["per_sm"] == 2 and d["nacc"] == 1 and base["small"] == 0
    assert _lib.debug_plan(12, 24, 256, 16384, 3, SMS)["MT"] == 1
    monkeypatch.setenv("WUNET_TC_OVR", "9:mt=1,ns=6")          # 6 splits of 48 columns would leave an empty split of 240
    with pytest.raises(_lib.WunetError, match="empty split"):
        _lib.debug_plan(12, 24, 256, 16384, 9, SMS)
    monkeypatch.setenv("WUNET_TC_OVR", "5:ns=1,small=1")       # 160 columns do not fit one consumer warpgroup's registers
    d = _lib.debug_plan(12, 24, 256, 16384, 5, SMS)
    assert d["Nh"] <= 64 and d["nsplit"] * d["Nh"] >= d["Npad"]


def test_unsupported_queries_fail_loudly():
    with pytest.raises(_lib.WunetError):
        _lib.debug_plan(12, 24, 256, 16384, 0, SMS)             # block 0 runs on CUDA cores (unless WUNET_TC_ENC0=1)
    with pytest.raises(_lib.WunetError):
        _lib.debug_plan(12, 20, 256, 16384, 3, SMS)             # channels_interval must be a multiple of 8
    with pytest.raises(_lib.WunetError):
        _lib.debug_plan(12, 24, 256, 1000, 3, SMS)              # T must be a multiple of 2^n_layers


def test_row_pair_and_group_modes(monkeypatch):
    """Block 1 runs over pairs of positions by default (9 taps, 48 -> 96 channels at half the rows); WUNET_TC_PAIR=0 gives the
    plain 15-tap block (the last block has no pair form), WUNET_TC_ENC0=1 a tensor-core plan for block 0 (groups of 8 samples)."""
    d = _lib.debug_plan(12, 24, 256, 16384, 1, SMS)
    assert (d["L"], d["Cin0"], d["Cout"], d["nchunks"], d["resident"]) == (4096, 48, 96, 1, 1)
    monkeypatch.setenv("WUNET_TC_PAIR", "0")
    d = _lib.debug_plan(12, 24, 256, 16384, 1, SMS)
    assert (d["L"], d["Cin0"], d["Cout"]) == (8192, 24, 48)
    assert _lib.debug_plan(12, 24, 256, 16384, 24, SMS)["Cout"] == 24
    monkeypatch.setenv("WUNET_TC_PAIR", "2")
    assert _lib.debug_plan(12, 24, 256, 16384, 24, SMS)["Cout"] == 24
    assert _lib.debug_plan(12, 24, 256, 16384, 1, SMS)["Cout"] == 48
    # frames too short for the pair form (fewer than 128 row pairs) keep the plain block
    monkeypatch.setenv("WUNET_TC_PAIR", "3")
    assert _lib.debug_plan(4, 8, 4, 256, 1, SMS)["Cout"] == 16
    monkeypatch.setenv("WUNET_TC_ENC0", "1")
    d = _lib.debug_plan(12, 24, 256, 16384, 0, SMS)
    assert (d["L"], d["Cin0"], d["Cout"], d["nchunks"], d["tg"]) == (2048, 8, 192, 1, 3)
