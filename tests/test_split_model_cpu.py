"""The fp32_tc / fp32 arithmetic model (tests/split_model.py) without a GPU: its split helpers, its distance from the pinned fp32
oracle, the size of the bugs its bars are there to see, and whether the GPU cases (tests/test_split_model_gpu.py) reach every
split-precision tiling the planner produces."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import split_model as sm
import test_split_model_gpu as gpu_cases
from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import _lib

ORACLE_TOL = 2e-5          # the model, not forced, against the oracle pinned to the reference's golden vectors


def bf16_half_ulp(hi):
    """half a bf16 ulp at |hi| (8 significant bits), float64"""
    return torch.exp2(torch.floor(torch.log2(hi.abs().clamp(min=1e-30))) - 8)


def random_fp32(n=200_000, seed=0):
    """fp32 values over many binades, both signs"""
    g = np.random.Generator(np.random.PCG64(seed))
    v = g.standard_normal(n) * np.exp2(g.integers(-30, 30, n))
    return torch.from_numpy(v.astype(np.float32)).double()


# ---------------------------------------------------------------------------------------------------------------------------
# the split helpers
# ---------------------------------------------------------------------------------------------------------------------------
def test_split_is_exact_in_fp32_and_within_2_to_the_minus_16():
    v = random_fp32()
    hi, lo = sm.split(v)
    s = hi + lo
    assert torch.equal(sm.f32(s), s), "hi + lo is not exact in fp32"
    assert torch.equal(sm.bf16_rn(hi), hi) and torch.equal(sm.bf16_rn(lo), lo), "a half is not a bf16 value"
    assert bool((lo.abs() <= bf16_half_ulp(hi)).all()), "|lo| above half an ulp of hi"
    assert bool(((s - v).abs() <= sm.SPLIT_REL * v.abs()).all()), "hi + lo further than 2^-16 from v"
    assert bool(((s - v).abs() > 2.0 ** -18 * v.abs()).any()), "lo is not rounded at all"


def test_halves_are_recovered_from_their_sum_up_to_ties():
    v = random_fp32(seed=1)
    hi, lo = sm.split(v)
    rh, rl = sm.recover(hi + lo)
    assert torch.equal(rh + rl, hi + lo)
    differ = (rh != hi)
    # only where |lo| is exactly half an ulp of hi (a midpoint of two bf16 values): the other hi, lo of the other sign, one
    # bf16 ulp between the two hi
    assert bool((lo[differ].abs() == bf16_half_ulp(hi[differ])).all())
    assert torch.equal(rl[differ], -lo[differ])
    assert bool(((rh - hi)[differ].abs() == 2 * bf16_half_ulp(hi[differ])).all())
    frac = float(differ.double().mean())
    assert 0 < frac < 0.005, frac                     # about 1 operand in 1000 (half of the ties, those with an odd hi)


def test_the_tie_case():
    """hi = 1 + 2^-7 (odd), v - hi just under half an ulp of hi: lo rounds up to 2^-8 exactly. The sum sits on the midpoint
    between 1 + 2^-7 and 1 + 2^-6, so recovery takes the even one. x_hi w_lo then moves by one bf16 ulp of x times |w_lo|,
    at most 2^-15 of |x w|."""
    v = torch.tensor([1 + 2.0 ** -7 + 2.0 ** -8 - 2.0 ** -20], dtype=torch.float64)
    hi, lo = sm.split(v)
    assert float(hi) == 1 + 2.0 ** -7 and float(lo) == 2.0 ** -8
    rh, rl = sm.recover(hi + lo)
    assert float(rh) == 1 + 2.0 ** -6 and float(rl) == -(2.0 ** -8)
    w = torch.tensor([1 + 2.0 ** -8 - 2.0 ** -16], dtype=torch.float64)        # |w_lo| near its largest, 2^-8 |w|
    w_hi, w_lo = sm.split(w)
    assert abs(float((rh - hi) * w_lo)) <= 2.0 ** -15 * float(v * w)


# ---------------------------------------------------------------------------------------------------------------------------
# the model against the pinned oracle
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", sm.MODES)
def test_model_matches_the_golden_small_config(golden_dir, mode):
    g = np.load(os.path.join(golden_dir, "small_n4_c8.npz"))
    n, ci, T, B = int(g["n_layers"]), int(g["channels_interval"]), int(g["T"]), int(g["B"])
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    x = wo.make_input(B, T, seed=int(g["input_seed"]))
    m = sm.forward_split_model(st, x, n, ci, mode)
    for i in range(2 * n + 1):
        assert np.abs(m.levels[i].numpy() - g[f"level_{i}"]).max() <= ORACLE_TOL, i
    assert np.abs(m.y.numpy() - g["y"]).max() <= ORACLE_TOL
    if mode == "fp32_tc":                           # and the split really rounds: the model is not the fp32 forward
        assert np.abs(m.levels[1].numpy() - g["level_1"]).max() > 1e-7


@pytest.mark.parametrize("mode", sm.MODES)
def test_model_matches_the_c_oracle_full_config(mode):
    n, ci = 12, 24
    st = wo.make_state(n, ci, seed=0)
    x = wo.make_input(1, 16384, seed=5)
    want_y, want = wo.COracle(n, ci).forward(st, x, return_levels=True)
    torch.set_num_threads(max(torch.get_num_threads(), 4))
    m = sm.forward_split_model(st, x, n, ci, mode)
    errs = [float(np.abs(m.levels[i].numpy() - want[i]).max()) for i in range(2 * n + 1)]
    assert max(errs) <= ORACLE_TOL, errs
    assert np.abs(m.y.numpy() - want_y).max() <= ORACLE_TOL


# ---------------------------------------------------------------------------------------------------------------------------
# sensitivity: the bugs the bars are for, evaluated in the model
# ---------------------------------------------------------------------------------------------------------------------------
SENS = (12, 24, 1, 4096, 0)


@pytest.fixture(scope="module")
def sens_model():
    n, ci, B, T, seed = SENS
    st = wo.make_state(n, ci, seed=seed)
    x = wo.make_input(B, T, seed=seed + 100)
    m = sm.forward_split_model(st, x, n, ci, "fp32_tc")
    return st, torch.from_numpy(x).double(), m


def mutated_block(st, xin, m, i, w_lo_zero=None, lo_times_w_lo=False, up_hi_only=False):
    """block i evaluated on the model's own stored levels with one K-loop mutation; -> stored value"""
    n, ci = SENS[0], SENS[1]
    prefix, _cin, _cout, k = wo.channel_plan(n, ci)[i]
    x, xh = sm.block_input(m.levels, i, n, "fp32_tc", xin, hi_only_up=up_hi_only)
    w = sm.weights(st, prefix)
    w_hi, w_lo = sm.split(w)
    if w_lo_zero is not None:
        w_lo = w_lo.clone()
        w_lo[:, w_lo_zero] = 0
    pad = (k - 1) // 2
    if lo_times_w_lo:                                             # lo data x w_lo in the slot of lo data x w_hi
        acc = F.conv1d(xh, w_hi, padding=pad) + F.conv1d(xh, w_lo, padding=pad) + F.conv1d(x - xh, w_lo, padding=pad)
    else:
        acc, _ = sm.products(x, xh, w, "fp32_tc", w_hi, w_lo)
    return sm.epilogue(acc, st, prefix, "fp32_tc")[0]


def worst(m, i, got):
    return float(sm.ratio((got - m.levels[i]).abs(), sm.block_bar(got, m.levels[i], m.scale[i], m.shift[i], "fp32_tc")).max())


N_S, CI_S = SENS[0], SENS[1]
CIN = {i: c for i, (_p, c, _o, _k) in enumerate(wo.channel_plan(N_S, CI_S))}
DEC = N_S + 1 + 4                                     # decoder 4: 216 upsampled + 192 skip channels
SKIP = wo.channel_plan(N_S, CI_S)[N_S - 1 - 4][2]
MUTATIONS = {
    "w_lo of the second 64-channel chunk zeroed (enc 6)": dict(i=6, w_lo_zero=slice(64, 128)),
    "w_lo of a decoder's skip chunks zeroed (dec 4)": dict(i=DEC, w_lo_zero=slice(CIN[DEC] - SKIP, CIN[DEC])),
    "lo data times w_lo (enc 3)": dict(i=3, lo_times_w_lo=True),
    "upsampled operand from hi only, window path (dec 9)": dict(i=N_S + 1 + 9, up_hi_only=True),
    "upsampled operand from hi only, per-row path (dec 2)": dict(i=N_S + 1 + 2, up_hi_only=True),
}


def test_the_unmutated_block_is_the_model(sens_model):
    st, xin, m = sens_model
    for i in (3, 6, DEC, 2 * N_S):
        assert torch.equal(mutated_block(st, xin, m, i), m.levels[i]), i


@pytest.mark.parametrize("name", list(MUTATIONS))
def test_bars_see_each_mutation_by_10x(sens_model, name):
    st, xin, m = sens_model
    kw = MUTATIONS[name]
    i = kw["i"]
    r = worst(m, i, mutated_block(st, xin, m, **kw))
    print(f"{name}: worst error/bar {r:.1f}")
    assert r >= 10, (name, r)


def test_bars_see_block_0_without_its_lo_store(sens_model):
    _st, _xin, m = sens_model
    r = worst(m, 0, sm.split(m.act[0])[0])
    print(f"block 0 stored without lo: worst error/bar {r:.1f}")
    assert r >= 10, r


def test_which_producer_path_the_mutations_take():
    """dec 9 reads a level of 2048 -> 4096 rows (the 8-row window), dec 2 one of 16 -> 32 rows (packed frames, per-row)"""
    T = SENS[3]
    assert T >> (N_S - 9) >= sm.PACKED_BELOW > T >> (N_S - 2)


# ---------------------------------------------------------------------------------------------------------------------------
# coverage: the GPU cases reach every split-precision feature the planner produces
# ---------------------------------------------------------------------------------------------------------------------------
SMS = 132                   # H100 SXM: the plan the cases run without WUNET_TC_SMS


def block0_form(ci, io16, enc0v):
    """Which kernel runs block 0 at fp32_tc, restated from the launch in wunet_tc.cu: the wide kernel for ci > 32, else the
    one-tile enc0_kernel for a 16-bit input or WUNET_TC_ENC0V=1, else the persistent enc0_kernel_v2 (float input, split
    mode). Block 0's form is not a plan field."""
    if ci > 32:
        return ("enc0", "wide")
    if io16 or enc0v == 1:
        return ("enc0", "one_tile")
    return ("enc0", "v2")


def features(d, i, n, ci, B):
    """the split-precision features one block plan exercises"""
    f = {("SP", 2 if (ci > 32 and d["nchunks"] > 48) else 1), ("nsplit", d["nsplit"])}
    if i > n:
        f.add("decoder_packed" if d["packed"] else "decoder_unpacked")
    f.add("resident" if d["resident"] else "weight_ring")
    per_cta = -(-d["m_tiles"] * d["nsplit"] // d["grid"])
    if per_cta >= 100:
        f.add("tiles_per_cta_ge_100")
    if per_cta == 1:
        f.add("one_tile_per_cta")
    if (d["packed"] and B % d["FR"] != 0) or (not d["packed"] and d["L"] % (128 * d["MT"]) != 0):
        f.add("partial_last_tile")
    return f


def plan_features(n, ci, B, T):
    out = set()
    for i in range(1, 2 * n + 1):
        out |= features(_lib.debug_plan(n, ci, B, T, i, SMS, "fp32_tc"), i, n, ci, B)
    return out


def universe():
    """the features over a sweep of plans and shapes"""
    out = set()
    for n, ci in [(4, 8), (6, 8), (5, 16), (5, 32), (12, 24), (12, 32), (10, 40), (12, 48), (12, 64)]:
        for B in (1, 2, 3, 5, 64, 256, 257):
            for T in {1 << n, 4 << n, 5 << (n + 2), 4096, 16384}:
                if T % (1 << n) == 0 and T >= 128:              # the tensor-core path needs frames of 128 samples
                    out |= plan_features(n, ci, B, T)
    return out


@pytest.fixture(autouse=True)
def _planner_defaults(monkeypatch):
    for k in ("WUNET_TC_SMS", "WUNET_TC_OVR", "WUNET_TC_GEMM", "WUNET_TC_MERGE", "WUNET_TC_PAIR"):
        monkeypatch.delenv(k, raising=False)


def test_the_planner_produces_the_named_features():
    u = universe()
    named = {("SP", 1), ("SP", 2), "decoder_packed", "decoder_unpacked", "resident", "weight_ring", ("nsplit", 1),
             "tiles_per_cta_ge_100", "one_tile_per_cta", "partial_last_tile"}
    assert named <= u, sorted(map(str, named - u))


def test_gpu_cases_reach_every_split_feature():
    required = universe() | {block0_form(40, False, 0), block0_form(24, True, 0), block0_form(24, False, 0)}
    got = set()
    for case in gpu_cases.CASES:
        n, ci, B, T = case.n, case.ci, case.B, case.T
        got |= plan_features(n, ci, B, T)
        got.add(block0_form(ci, case.half, case.enc0v))
    missing = sorted(map(str, required - got))
    assert not missing, f"no fp32_tc GPU case reaches {missing}"


def test_gpu_case_picks_are_in_the_batch():
    for case in gpu_cases.CASES + gpu_cases.FP32_CASES:
        assert case.pick is None or max(case.pick) < case.B, case.name
