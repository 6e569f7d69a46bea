"""GPU parity tests (pytest -m gpu, on an H100). The CUDA path is called through the C ABI
(via the drop-in module's ctypes shim) and compared with the oracle and the committed golden vectors
generated from the live reference module."""
import os

import numpy as np
import pytest
import torch

from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model, _lib

pytestmark = pytest.mark.gpu

FP32_TOL = 1e-4     # BASELINE.json north_star: <= 1e-4 max-abs fp32 vs the reference forward


def make_model(n, ci, st, precision):
    m = Model(n, ci, precision=precision)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    return m.to("cuda:0").eval()


def run(m, x):
    with torch.no_grad():
        y = m(torch.from_numpy(x).to("cuda:0"))
    torch.cuda.synchronize()
    return y.cpu().numpy()


@pytest.fixture(scope="module")
def full(golden_dir):
    return np.load(os.path.join(golden_dir, "full_n12_c24_b2.npz"))


@pytest.fixture(scope="module")
def state_full():
    return wo.make_state(12, 24, seed=0)


def test_extension_is_loaded_not_a_fallback():
    lib = _lib.load()
    assert b"sm_90a" in lib.wunet_version()
    assert torch.cuda.get_device_capability(0) == (9, 0)


def test_fp32_small_config_all_levels(golden_dir):
    g = np.load(os.path.join(golden_dir, "small_n4_c8.npz"))
    n, ci, T, B = int(g["n_layers"]), int(g["channels_interval"]), int(g["T"]), int(g["B"])
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    x = wo.make_input(B, T, seed=int(g["input_seed"]))
    m = make_model(n, ci, st, "fp32")
    y = run(m, x)
    for i in range(2 * n + 1):
        lv = m.read_level(i, B, T).cpu().numpy()
        assert lv.shape == g[f"level_{i}"].shape
        assert np.abs(lv - g[f"level_{i}"]).max() <= FP32_TOL, f"level {i}"
    assert np.abs(y - g["y"]).max() <= FP32_TOL


def test_fp32_full_config_vs_golden_and_oracle(full, state_full):
    x = wo.make_input(2, 16384, seed=int(full["input_seed"]))
    m = make_model(12, 24, state_full, "fp32")
    y = run(m, x)
    for i in range(25):
        lv = m.read_level(i, 2, 16384).cpu().numpy()
        idx = full[f"probe_idx_{i}"]
        err = np.abs(lv[0][:, idx] - full[f"probe_{i}"]).max()
        assert err <= FP32_TOL, f"level {i}: {err}"
        a = np.abs(lv.astype(np.float64)).sum()
        assert abs(a - float(full[f"abssum_{i}"])) <= 1e-5 * a + 1e-2, f"level {i} abssum"
    err = np.abs(y - full["y"]).max()
    assert err <= FP32_TOL, err
    assert m.last_launch_count() == 26


def test_fp32_config2_batch64_vs_oracle_subset(state_full):
    """BASELINE.json configs[1]: B=64, T=16384 fp32, <= 1e-4. The oracle checks 4 of the 64 frames in full
    (frames are independent in eval mode); batch-permutation invariance covers the rest."""
    B = 64
    x = wo.make_input(B, 16384, seed=4321)
    m = make_model(12, 24, state_full, "fp32")
    y = run(m, x)
    pick = [0, 17, 42, 63]
    want = wo.COracle(12, 24).forward(state_full, x[pick])
    assert np.abs(y[pick] - want).max() <= FP32_TOL
    perm = np.random.default_rng(0).permutation(B)
    y2 = run(m, x[perm])
    assert np.array_equal(y2, y[perm]), "eval forward must be batch-permutation invariant, bit for bit"
    assert np.isfinite(y).all() and np.abs(y).max() < 1.0


def test_fp32_edge_vectors(golden_dir, state_full):
    g = np.load(os.path.join(golden_dir, "edges_n12_c24.npz"))
    m = make_model(12, 24, state_full, "fp32")
    for name, xe in wo.edge_inputs(16384).items():
        assert np.abs(run(m, xe) - g[name]).max() <= FP32_TOL, name
    for Tx in (4096, 20480):
        y = run(m, wo.make_input(1, Tx, seed=77 + Tx))
        assert np.abs(y - g[f"T{Tx}"]).max() <= FP32_TOL, Tx


def test_fp32_b1_loop_equals_batched(state_full):
    """enhancement.py:64-66 forwards one chunk at a time; stacking chunks on the batch axis is equivalent."""
    x = wo.make_input(3, 16384, seed=99)
    m = make_model(12, 24, state_full, "fp32")
    yb = run(m, x)
    for b in range(3):
        assert np.abs(run(m, x[b:b + 1]) - yb[b:b + 1]).max() <= 1e-6


def test_bad_length_raises(state_full):
    m = make_model(12, 24, state_full, "fp32")
    with pytest.raises(_lib.WunetError, match="multiple of 2"):
        m(torch.zeros(1, 1, 16000, device="cuda:0"))


def test_weight_cache_invalidation(state_full):
    m = make_model(12, 24, state_full, "fp32")
    x = wo.make_input(1, 4096, seed=5)
    y0 = run(m, x)
    with torch.no_grad():
        m.out[0].bias.add_(0.25)                      # in-place update bumps _version (optimizer.step does this)
    y1 = run(m, x)
    assert np.abs(y1 - y0).max() > 1e-3
    st2 = wo.make_state(12, 24, seed=5)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st2.items()})
    y2 = run(m, x)
    assert np.abs(y2 - wo.COracle().forward(st2, x)).max() <= FP32_TOL
    m.cpu(); m.to("cuda:0")                           # base_trainer.py:103-124 does this around checkpointing
    assert np.array_equal(run(m, x), y2)


def test_forward_host_matches_device_path(state_full):
    m = make_model(12, 24, state_full, "fp32")
    x = wo.make_input(4, 16384, seed=8)
    xh = torch.from_numpy(x).pin_memory()
    yh = m.forward_host(xh)
    assert np.array_equal(yh.numpy(), run(m, x))


# ---- bf16 tensor-core path (BASELINE.json configs[2]) -------------------------------------------------------
# Every activation is stored in bf16 (8 mantissa bits: relative rounding 2^-9 = 0.2 %) and every conv uses bf16
# operands with fp32 accumulation, so the per-level bound is relative to the level's dynamic range:
BF16_LEVEL_REL = 8e-3       # max-abs(level error) / max-abs(level) ; measured 0.3-0.5 %
BF16_OUT_TOL = 2e-3         # max-abs on the tanh output (|y| <= 0.35 here); measured 6e-4 (SURVEY §8c: ~2e-3 for bf16 operands)


def bf16_model(n, ci, st, store_last=False):
    """store_last=False is the benchmarked variant (last decoder block fused with the head, never stored); True also
    materialises that block so that read_level(2n) works (the flag is read when the library creates the model's context)."""
    os.environ["WUNET_TC_STORE_LAST"] = "1" if store_last else "0"
    return make_model(n, ci, st, "bf16")


def test_bf16_small_config_all_levels(golden_dir):
    g = np.load(os.path.join(golden_dir, "small_n4_c8.npz"))
    n, ci, T, B = int(g["n_layers"]), int(g["channels_interval"]), int(g["T"]), int(g["B"])
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    x = wo.make_input(B, T, seed=int(g["input_seed"]))
    m = bf16_model(n, ci, st, store_last=True)
    y = run(m, x)
    for i in range(2 * n + 1):
        lv = m.read_level(i, B, T).cpu().numpy()
        ref = g[f"level_{i}"]
        assert np.abs(lv - ref).max() <= BF16_LEVEL_REL * np.abs(ref).max(), f"level {i}"
    assert np.abs(y - g["y"]).max() <= BF16_OUT_TOL
    y_fused = run(bf16_model(n, ci, st), x)                  # the variant that is benchmarked: head fused, no store
    assert np.array_equal(y_fused, y)


def test_bf16_full_config_all_levels_vs_oracle(full, state_full):
    x = wo.make_input(2, 16384, seed=int(full["input_seed"]))
    want, levels = wo.COracle(12, 24).forward(state_full, x, return_levels=True)
    m = bf16_model(12, 24, state_full, store_last=True)
    y = run(m, x)
    rels = []
    for i in range(25):
        lv = m.read_level(i, 2, 16384).cpu().numpy()
        err = np.abs(lv - levels[i]).max()
        rels.append(float(err / np.abs(levels[i]).max()))
        assert err <= BF16_LEVEL_REL * np.abs(levels[i]).max(), f"level {i}: {err}"
    print("bf16 per-level relative errors: " + " ".join("%.4f" % r for r in rels))
    print("bf16 output max-abs error vs oracle: %.3e" % np.abs(y - want).max())
    assert np.abs(y - full["y"]).max() <= BF16_OUT_TOL
    assert np.abs(y - want).max() <= BF16_OUT_TOL
    assert m.last_launch_count() == 25          # enc0 + 24 fused conv blocks (head fused into the last one)
    m2 = bf16_model(12, 24, state_full)         # benchmarked variant: no store of the last block
    y2 = run(m2, x)
    assert np.array_equal(y2, y)
    with pytest.raises(_lib.WunetError, match="not materialised"):
        m2.read_level(24, 2, 16384)


def test_bf16_odd_shapes_vs_oracle(state_full):
    """T = 4096 (bottom of the U down to L = 1) and 20480 (tile counts not powers of two), batch 5."""
    for T, B in ((4096, 5), (20480, 3)):
        x = wo.make_input(B, T, seed=100 + T)
        want = wo.COracle(12, 24).forward(state_full, x)
        m = bf16_model(12, 24, state_full)
        assert np.abs(run(m, x) - want).max() <= BF16_OUT_TOL, T


def test_bf16_config3_batch256_properties(state_full):
    """BASELINE.json configs[2] size (B=256), the benchmarked kernel variant (head fused, last block not stored):
    16 oracle-checked frames spread over the batch + batch-permutation invariance (bit exact)."""
    B = 256
    x = wo.make_input(B, 16384, seed=2468)
    m = bf16_model(12, 24, state_full)
    y = run(m, x)
    pick = [0, 1, 17, 31, 64, 100, 127, 128, 129, 150, 177, 200, 222, 240, 254, 255]
    want = wo.COracle(12, 24).forward(state_full, x[pick])
    err = float(np.abs(y[pick] - want).max())
    print("bf16 B=256 (benchmarked variant): max-abs error over 16 frames %.3e" % err)
    assert err <= BF16_OUT_TOL
    perm = np.random.default_rng(1).permutation(B)
    assert np.array_equal(run(m, x[perm]), y[perm])
    # the tiling depends on the batch (column splits, grids), the K-loop order, hence every output bit, must not. (Batches below
    # 64 frames take the packed-frame kernels instead of the
    # dense GEMM for the blocks of at most 16 samples - different arithmetic for the folded interpolation, so they are compared
    # among themselves.)
    assert np.array_equal(run(m, x[:64]), y[:64])
    assert np.array_equal(run(m, x[:3]), run(m, x[:5])[:3])
    assert np.isfinite(y).all() and np.abs(y).max() < 1.0


def test_bf16_large_ragged_batch_and_long_frames(state_full):
    """Sizes past the benchmark's: a batch of 1000 frames (no multiple of any tile / packing factor; 12 GB workspace) and
    frames of 65536 samples (4x the reference's sample_length: 4x the tiles per frame on every level). Oracle-checked frames
    + agreement with the same frames run in a batch of 256 (bit exact: batches >= 64 share their K-loop order)."""
    B = 1000
    x = wo.make_input(B, 16384, seed=4321)
    m = bf16_model(12, 24, state_full)
    y = run(m, x)
    assert y.shape == (B, 1, 16384) and np.isfinite(y).all()
    pick = [0, 255, 256, 511, 777, 998, 999]
    want = wo.COracle(12, 24).forward(state_full, x[pick])
    assert np.abs(y[pick] - want).max() <= BF16_OUT_TOL
    assert np.array_equal(run(m, x[744:1000]), y[744:1000])
    T = 65536
    xl = wo.make_input(3, T, seed=97)
    yl = run(m, xl)
    wantl = wo.COracle(12, 24).forward(state_full, xl[1:2])
    assert np.abs(yl[1:2] - wantl).max() <= BF16_OUT_TOL
    assert np.array_equal(run(m, xl[[2, 0, 1]]), yl[[2, 0, 1]])


def test_bf16_edge_vectors(golden_dir, state_full):
    g = np.load(os.path.join(golden_dir, "edges_n12_c24.npz"))
    m = bf16_model(12, 24, state_full)
    for name, xe in wo.edge_inputs(16384).items():
        assert np.abs(run(m, xe) - g[name]).max() <= BF16_OUT_TOL, name


def test_bf16_forward_host_matches_device_path(state_full):
    m = bf16_model(12, 24, state_full)
    x = wo.make_input(8, 16384, seed=8)
    yh = m.forward_host(torch.from_numpy(x).pin_memory())
    assert np.array_equal(yh.numpy(), run(m, x))


# ---- fp32_tc: fp32-grade results on the tensor cores (bf16 hi + lo split, three MMAs per product) -----------------------
# The tensor cores AND <= 1e-4 on the same path: every fp32 parity case again, same tolerance.
def test_fp32_tc_small_config_all_levels(golden_dir):
    g = np.load(os.path.join(golden_dir, "small_n4_c8.npz"))
    n, ci, T, B = int(g["n_layers"]), int(g["channels_interval"]), int(g["T"]), int(g["B"])
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    x = wo.make_input(B, T, seed=int(g["input_seed"]))
    os.environ["WUNET_TC_STORE_LAST"] = "1"
    m = make_model(n, ci, st, "fp32_tc")
    y = run(m, x)
    errs = []
    for i in range(2 * n + 1):
        lv = m.read_level(i, B, T).cpu().numpy()
        errs.append(float(np.abs(lv - g[f"level_{i}"]).max()))
    print("fp32_tc small config: per-level max-abs errors " + " ".join("%.1e" % e for e in errs) + " | output %.2e" % np.abs(y - g["y"]).max())
    assert max(errs) <= FP32_TOL, errs
    assert np.abs(y - g["y"]).max() <= FP32_TOL


def test_fp32_tc_full_config_vs_golden_and_oracle(full, state_full):
    x = wo.make_input(2, 16384, seed=int(full["input_seed"]))
    os.environ["WUNET_TC_STORE_LAST"] = "1"
    m = make_model(12, 24, state_full, "fp32_tc")
    y = run(m, x)
    errs = []
    for i in range(25):
        lv = m.read_level(i, 2, 16384).cpu().numpy()
        idx = full[f"probe_idx_{i}"]
        errs.append(float(np.abs(lv[0][:, idx] - full[f"probe_{i}"]).max()))
    err = float(np.abs(y - full["y"]).max())
    print("fp32_tc full config: per-level probe errors " + " ".join("%.1e" % e for e in errs) + " | output %.2e" % err)
    assert max(errs) <= FP32_TOL, errs
    assert err <= FP32_TOL, err
    assert m.last_launch_count() == 25
    os.environ["WUNET_TC_STORE_LAST"] = "0"
    assert np.array_equal(run(make_model(12, 24, state_full, "fp32_tc"), x), y)       # head fused, last block not stored


def test_fp32_tc_config2_batch64_edges_and_odd_lengths(golden_dir, state_full):
    os.environ["WUNET_TC_STORE_LAST"] = "0"
    m = make_model(12, 24, state_full, "fp32_tc")
    B = 64
    x = wo.make_input(B, 16384, seed=4321)
    y = run(m, x)
    pick = [0, 17, 42, 63]
    want = wo.COracle(12, 24).forward(state_full, x[pick])
    err = float(np.abs(y[pick] - want).max())
    print("fp32_tc B=64: max-abs error over 4 frames %.2e" % err)
    assert err <= FP32_TOL
    perm = np.random.default_rng(0).permutation(B)
    assert np.array_equal(run(m, x[perm]), y[perm])
    g = np.load(os.path.join(golden_dir, "edges_n12_c24.npz"))
    for name, xe in wo.edge_inputs(16384).items():
        assert np.abs(run(m, xe) - g[name]).max() <= FP32_TOL, name
    for Tx in (4096, 20480):
        assert np.abs(run(m, wo.make_input(1, Tx, seed=77 + Tx)) - g[f"T{Tx}"]).max() <= FP32_TOL, Tx
    yh = m.forward_host(torch.from_numpy(x[:8]).pin_memory())
    assert np.array_equal(yh.numpy(), run(m, x[:8]))


# ---- row-pair / row-group forms of the narrow blocks (DESIGN.md 5.1): every switch position against the oracle ------------
@pytest.mark.parametrize("pair,enc0_tc", [("0", "0"), ("1", "0"), ("0", "1")])
def test_bf16_row_pair_and_group_forms_vs_oracle(state_full, pair, enc0_tc, monkeypatch):
    """WUNET_TC_PAIR bit 0 (block 1 over pairs of positions: the default; 0 = the plain block), WUNET_TC_ENC0=1
    (block 0 on the tensor cores over groups of 8 samples): the same operator, so the same bounds as the plain blocks hold - per
    block against the oracle's activations, on the output, with impulses at both frame edges (zero padding of the row-pair rows,
    end points of the upsampling) - and the benchmarked variant (last block not stored) gives the same output."""
    monkeypatch.setenv("WUNET_TC_PAIR", pair)
    monkeypatch.setenv("WUNET_TC_ENC0", enc0_tc)
    B, T = 2, 16384
    x = wo.make_input(B, T, seed=4321)
    x[1, 0, 0] += 0.9
    x[1, 0, T - 1] -= 0.9
    want, levels = wo.COracle(12, 24).forward(state_full, x, return_levels=True)
    m = bf16_model(12, 24, state_full, store_last=True)
    y = run(m, x)
    assert m.last_launch_count() == (26 if enc0_tc == "1" else 25)
    for i in (0, 1, 2, 23, 24):
        lv = m.read_level(i, B, T).cpu().numpy()
        err = np.abs(lv - levels[i]).max()
        assert err <= BF16_LEVEL_REL * np.abs(levels[i]).max(), f"block {i}: {err}"
    assert np.abs(y - want).max() <= BF16_OUT_TOL
    m._release()
    y2 = run(bf16_model(12, 24, state_full), x)
    assert np.array_equal(y2, y)
    # a short-frame network where the forms do not apply (fewer than 128 row pairs / 1024 samples): plain blocks, still correct
    st = wo.make_state(4, 8, seed=3)
    xs = wo.make_input(3, 256, seed=9)
    ms = bf16_model(4, 8, st)
    assert np.abs(run(ms, xs) - wo.COracle(4, 8).forward(st, xs)).max() <= BF16_OUT_TOL


def test_enc0_persistent_form_is_bit_identical(state_full, monkeypatch):
    """The two CUDA-core forms of block 0 (WUNET_TC_ENC0V=1: one tile per block, 2: persistent blocks with cp.async prefetch) run
    the same arithmetic in the same order, also for frames that are not a multiple of the 1024-sample tile."""
    outs = {}
    for v in ("1", "2"):
        monkeypatch.setenv("WUNET_TC_ENC0V", v)
        m = bf16_model(12, 24, state_full, store_last=True)
        x = wo.make_input(3, 16384, seed=77)
        y = run(m, x)
        b0 = m.read_level(0, 3, 16384).cpu().numpy()
        m._release()
        st = wo.make_state(4, 8, seed=2)
        ms = make_model(4, 8, st, "fp32_tc")
        ys = run(ms, wo.make_input(5, 2064, seed=6))
        ms._release()
        outs[v] = (y, b0, ys)
    for a, b in zip(outs["1"], outs["2"]):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("n,ci,B,T", [(5, 32, 3, 4096), (5, 16, 2, 4096), (6, 8, 3, 2048), (5, 32, 130, 1024)])
def test_bf16_other_channel_plans_vs_oracle(n, ci, B, T):
    """Channel plans other than the reference's 24 base filters (block 1 in row-pair form: 2 x ci = 16 .. 64 virtual input
    channels, one K chunk; the last case at a batch that takes the swept tiling): output and block 1 against the oracle."""
    st = wo.make_state(n, ci, seed=1)
    x = wo.make_input(B, T, seed=2)
    want, levels = wo.COracle(n, ci).forward(st, x, return_levels=True)
    m = bf16_model(n, ci, st, store_last=True)
    y = run(m, x)
    b1 = m.read_level(1, B, T).cpu().numpy()
    assert np.abs(b1 - levels[1]).max() <= BF16_LEVEL_REL * np.abs(levels[1]).max()
    assert np.abs(y - want).max() <= BF16_OUT_TOL
