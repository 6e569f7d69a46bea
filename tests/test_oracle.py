"""Pins the oracle (oracle/wunet_oracle.{c,py}) against golden vectors produced by the live
reference module (oracle/gen_golden.py -> tests/golden/).  CPU only."""
import json
import os

import numpy as np
import pytest

from oracle import wunet_oracle as wo

ORACLE_TOL = 2e-5   # oracle (double accumulate) vs reference fp32 CPU forward; measured ~2e-6


@pytest.fixture(scope="module")
def small(golden_dir):
    return np.load(os.path.join(golden_dir, "small_n4_c8.npz"))


@pytest.fixture(scope="module")
def full(golden_dir):
    return np.load(os.path.join(golden_dir, "full_n12_c24_b2.npz"))


@pytest.fixture(scope="module")
def edges(golden_dir):
    return np.load(os.path.join(golden_dir, "edges_n12_c24.npz"))


def test_state_dict_surface_matches_reference(golden_dir):
    surf = json.load(open(os.path.join(golden_dir, "state_dict_surface.json")))
    ref = [(k, tuple(s), d) for k, s, d in surf["state_dict"]]
    assert ref == wo.state_keys(12, 24)
    assert len(ref) == 177
    assert surf["n_params"] == 10132802
    n_float = sum(int(np.prod(s)) for _k, s, d in ref if d == "float32")
    assert wo.COracle(12, 24).lib.wunet_oracle_param_count(12, 24) == n_float


@pytest.mark.parametrize("impl", ["numpy", "c"])
def test_small_config_all_levels(small, impl):
    n, ci, T, B = int(small["n_layers"]), int(small["channels_interval"]), int(small["T"]), int(small["B"])
    st = wo.make_state(n, ci, seed=int(small["state_seed"]))
    x = wo.make_input(B, T, seed=int(small["input_seed"]))
    if impl == "numpy":
        y, levels = wo.forward_numpy(st, x, n, ci, return_levels=True)
    else:
        y, levels = wo.COracle(n, ci).forward(st, x, return_levels=True)
    assert len(levels) == 2 * n + 1
    for i, lv in enumerate(levels):
        ref = small[f"level_{i}"]
        assert lv.shape == ref.shape
        assert np.abs(lv - ref).max() <= ORACLE_TOL, f"level {i}"
    assert np.abs(y - small["y"]).max() <= ORACLE_TOL


def test_full_config_c_oracle(full):
    n, ci, T, B = 12, 24, 16384, 2
    st = wo.make_state(n, ci, seed=int(full["state_seed"]))
    x = wo.make_input(B, T, seed=int(full["input_seed"]))
    y, levels = wo.COracle(n, ci).forward(st, x, return_levels=True)
    err = np.abs(y - full["y"]).max()
    assert err <= ORACLE_TOL, err
    for i, lv in enumerate(levels):
        idx = full[f"probe_idx_{i}"]
        assert np.abs(lv[0][:, idx] - full[f"probe_{i}"]).max() <= ORACLE_TOL, f"level {i}"
        s = lv.astype(np.float64).sum()
        a = np.abs(lv.astype(np.float64)).sum()
        assert abs(a - float(full[f"abssum_{i}"])) <= 1e-6 * a + 1e-3, f"level {i} abssum"
        assert abs(s - float(full[f"sum_{i}"])) <= 1e-6 * a + 1e-3, f"level {i} sum"


def test_numpy_and_c_agree_full_b1():
    st = wo.make_state(12, 24, seed=3)
    x = wo.make_input(1, 4096, seed=4)
    y0 = wo.forward_numpy(st, x)
    y1 = wo.COracle().forward(st, x)
    assert np.abs(y0 - y1).max() <= 2e-6


def test_edge_vectors(edges):
    st = wo.make_state(12, 24, seed=int(edges["state_seed"]))
    orc = wo.COracle()
    for name, xe in wo.edge_inputs(16384).items():
        y = orc.forward(st, xe)
        assert np.abs(y - edges[name]).max() <= ORACLE_TOL, name
    for Tx in (4096, 20480):
        y = orc.forward(st, wo.make_input(1, Tx, seed=77 + Tx))
        assert np.abs(y - edges[f"T{Tx}"]).max() <= ORACLE_TOL, Tx


def test_bad_length_raises():
    st = wo.make_state(12, 24, seed=0)
    with pytest.raises(ValueError):
        wo.COracle().forward(st, wo.make_input(1, 16000))
    with pytest.raises(ValueError):
        wo.forward_numpy(st, wo.make_input(1, 16000))


def test_torch_port_matches_golden(full):
    import torch
    st = wo.make_state(12, 24, seed=int(full["state_seed"]))
    x = wo.make_input(2, 16384, seed=int(full["input_seed"]))
    st_t = {k: torch.from_numpy(v) for k, v in st.items()}
    with torch.no_grad():
        y = wo.torch_port_forward(st_t, torch.from_numpy(x)).numpy()
    assert np.abs(y - full["y"]).max() <= 1e-6


def test_batch_independence():
    """eval-mode frames are independent: batched == per-frame (SURVEY §3.2)."""
    st = wo.make_state(12, 24, seed=0)
    x = wo.make_input(2, 4096, seed=9)
    orc = wo.COracle()
    yb = orc.forward(st, x)
    y0 = orc.forward(st, x[0:1])
    y1 = orc.forward(st, x[1:2])
    assert np.array_equal(yb[0:1], y0) and np.array_equal(yb[1:2], y1)


def test_bf16_arithmetic_model_sits_where_the_gpu_path_was_measured(golden_dir):
    """oracle/wunet_bf16_model.py restates the bf16 path's roundings; against the fp32 golden vectors it must show the
    distance the CUDA path is held to (test_parity_gpu.py: 0.8 % of each level's range, 2e-3 on the output), not more."""
    from oracle import wunet_bf16_model as wb
    g = np.load(os.path.join(golden_dir, "small_n4_c8.npz"))
    n, ci, T, B = int(g["n_layers"]), int(g["channels_interval"]), int(g["T"]), int(g["B"])
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    x = wo.make_input(B, T, seed=int(g["input_seed"]))
    y, levels = wb.forward_bf16_model(st, x, n, ci, return_levels=True)
    assert np.abs(y - g["y"]).max() <= 5e-3
    for i, lv in enumerate(levels):
        ref = g[f"level_{i}"]
        assert lv.shape == ref.shape
        assert np.abs(lv - ref).max() <= 1.5e-2 * np.abs(ref).max(), i
    # and it is a different function from the fp32 forward: the roundings are really applied
    assert np.abs(levels[1] - g["level_1"]).max() > 1e-5
