"""The GPU checks of the tensor-core tiling (tests/test_bf16_model_gpu.py, tests/test_bf16_tiling_gpu.py) only mean something if
their cases reach the tilings that can go wrong. This guard enumerates the plans of their case tables with the host-only
planner query (no GPU needed) and requires that together they reach:

- weights resident in shared memory, and a streamed weight ring whose stages hold fewer taps than the kernel (tg < KS);
- 1, 2 and at least 3 column splits;
- packed tiles of one frame, of several frames, and of the whole batch;
- input rings 2 and 3 deep (the planner never produces a single input stage, na = 1, so that one is not required);
- the small (two CTAs per SM) flavour on an encoder and on a decoder;
- a decoder with the merged tail chunk, and block 1 in row-pair form;
- every column tile Nh of the dense GEMM that the planner produces for some shape and SM count, and a GEMM whose last
  128-frame row tile is partial;
- a persistent block with at least 100 tiles per CTA, and one with a single tile per CTA.

It fails as soon as a change of the case tables or of the planner drops one of them."""
import pytest

import test_bf16_model_gpu as model_cases
import test_bf16_tiling_gpu as tiling_cases
from wave_u_net_for_speech_enhancement_b200 import _lib

SMS = 132                   # H100 SXM: the plan the cases run without WUNET_TC_SMS

REQUIRED = {
    "resident", "weight_ring_tg_lt_ks", ("nsplit", 1), ("nsplit", 2), ("nsplit", ">=3"),
    "packed_fr1", "packed_fr_gt1", "packed_fr_eq_batch", ("na", 2), ("na", 3), "small_encoder", "small_decoder",
    "merged_tail", "row_pair_block1", "gemm_partial_row_tile", "tiles_per_cta_ge_100", "one_tile_per_cta",
}


def plan_queries():
    """(n, ci, B, T, sms, precision, WUNET_TC_OVR) of every plan the GPU cases run."""
    q = []
    for n, ci, B, T, _seed in model_cases.MODEL_CASES:
        q.append((n, ci, B, T, SMS, "bf16", None))
        if B == 256:
            q.append((n, ci, B, T, model_cases.OTHER_SMS, "bf16", None))
    n, ci, B, T, _seed = model_cases.FP32_TC_CASE
    q.append((n, ci, B, T, SMS, "fp32_tc", None))
    for n, ci, B, T, sms in tiling_cases.SMS_CASES:
        for p in tiling_cases.PRECISIONS:
            q += [(n, ci, B, T, SMS, p, None), (n, ci, B, T, sms, p, None)]
    n, ci, B, T = tiling_cases.OVR_SHAPE
    q += [(n, ci, B, T, SMS, "bf16", ovr) for _blk, ovr in tiling_cases.OVR_CASES]
    for n, ci, B, T, p, sms in tiling_cases.HOST_CASES:
        q.append((n, ci, B, T, sms or SMS, p, None))
    return q


def features(d, i, n, ci, B, precision):
    """The tiling features one block plan exercises."""
    if d["small"] == 2:                                  # dense GEMM over frames: one 128-frame x Nh tile per CTA
        f = {("gemm_nh", d["Nh"])}
        if d["m_tiles"] >= 2 and B % 128 != 0:
            f.add("gemm_partial_row_tile")
        return f
    dec = i > n
    f = {("nsplit", d["nsplit"] if d["nsplit"] < 3 else ">=3"), ("na", d["na"])}
    if d["resident"]:
        f.add("resident")
    elif d["ngroups"] > 1:
        f.add("weight_ring_tg_lt_ks")
    if d["packed"]:
        f.add("packed_fr1" if d["FR"] == 1 else "packed_fr_gt1")
        if d["FR"] == B and B > 1:
            f.add("packed_fr_eq_batch")
    if d["small"] == 1:
        f.add("small_decoder" if dec else "small_encoder")
    if precision == "bf16" and dec and d["nchunks"] == -(-d["Cin0"] // 64) + -(-d["Cin1"] // 64) - 1:
        f.add("merged_tail")                             # [skip tail | upsampled tail] share one 64-channel chunk
    if precision == "bf16" and i == 1 and d["Cout"] == 4 * ci:
        f.add("row_pair_block1")                         # pairs of positions: twice block 1's 2 ci output channels
    per_cta = -(-d["m_tiles"] * d["nsplit"] // d["grid"])
    if per_cta >= 100:
        f.add("tiles_per_cta_ge_100")
    if per_cta == 1:
        f.add("one_tile_per_cta")
    return f


def reached(queries, monkeypatch):
    got = set()
    for n, ci, B, T, sms, precision, ovr in queries:
        if ovr is None:
            monkeypatch.delenv("WUNET_TC_OVR", raising=False)
        else:
            monkeypatch.setenv("WUNET_TC_OVR", ovr)
        for i in range(1, 2 * n + 1):
            got |= features(_lib.debug_plan(n, ci, B, T, i, sms, precision), i, n, ci, B, precision)
    return got


def gemm_nh_the_planner_produces():
    """Column tiles of the dense GEMM over a grid of shapes (like test_plan_cpu's) and every SM count from 1 to 132."""
    out = set()
    for n, ci in [(4, 8), (8, 16), (12, 24), (12, 32), (12, 8), (10, 24)]:
        for B in (64, 128, 256, 1000):                   # the GEMM needs a batch of at least 64 frames
            for T in {1 << n, 4 << n, 16384 if 16384 % (1 << n) == 0 else 8 << n}:
                if T < 128:
                    continue
                blocks = [i for i in range(1, 2 * n) if ((T >> i) if i <= n else (T >> (2 * n - i))) <= 16]
                for sms in range(1, SMS + 1):
                    for i in blocks:
                        d = _lib.debug_plan(n, ci, B, T, i, sms)
                        if d["small"] == 2:
                            out.add(d["Nh"])
    return out


@pytest.fixture(autouse=True)
def _planner_defaults(monkeypatch):
    for k in tiling_cases.PLAN_KNOBS:
        monkeypatch.delenv(k, raising=False)


def test_gpu_cases_reach_every_tiling_feature(monkeypatch):
    got = reached(plan_queries(), monkeypatch)
    assert REQUIRED <= got, f"no GPU case reaches {sorted(map(str, REQUIRED - got))}"


def test_gpu_cases_reach_every_gemm_column_tile(monkeypatch):
    universe = gemm_nh_the_planner_produces()
    assert universe == set(range(16, 129, 16)), universe
    got = {f[1] for f in reached(plan_queries(), monkeypatch) if isinstance(f, tuple) and f[0] == "gemm_nh"}
    assert universe <= got, f"GEMM column tiles Nh {sorted(universe - got)} are never run on the GPU"


def test_override_cases_are_accepted_and_change_their_block(monkeypatch):
    """Every WUNET_TC_OVR case is a plan the planner accepts, differs from the default plan of its block and leaves the other
    blocks alone; every key is exercised on some block."""
    n, ci, B, T = tiling_cases.OVR_SHAPE
    base = [_lib.debug_plan(n, ci, B, T, i, SMS) for i in range(1, 2 * n + 1)]
    keys = set()
    for blk, ovr in tiling_cases.OVR_CASES:
        monkeypatch.setenv("WUNET_TC_OVR", ovr)
        got = [_lib.debug_plan(n, ci, B, T, i, SMS) for i in range(1, 2 * n + 1)]
        assert [i + 1 for i in range(2 * n) if got[i] != base[i]] == [blk], ovr
        kv = ovr.split(":", 1)[1]
        keys.add("ns+1" if kv.startswith("ns=") else kv)
    assert set(tiling_cases.OVR_KEYS) <= keys, keys
