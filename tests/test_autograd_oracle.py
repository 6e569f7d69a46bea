"""Autograd oracle: the float64 restatement in oracle/wunet_autograd_oracle.py (input gradient; BatchNorm in training and in
eval mode) against the vectors produced by autograd on the live reference module with x.requires_grad_(True)
(oracle/gen_golden_autograd.py), and the training-mode vectors against the existing training goldens. CPU only."""
import os

import numpy as np
import pytest

from oracle import wunet_autograd_oracle as wa
from oracle import wunet_oracle as wo

REL = 1e-9           # both sides are float64; differences are summation order only
SAME = 1e-12         # the same float64 computation on both sides (only the input now requires grad)


def make_pair(B, T, seed):
    g = np.random.Generator(np.random.PCG64(seed))
    clean = (0.1 * g.standard_normal((B, 1, T))).astype(np.float32)
    noisy = (clean + 0.05 * g.standard_normal((B, 1, T))).astype(np.float32)
    return noisy, clean


def rel_err(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def noise_only(k, mode):
    """A conv bias ahead of a training-mode BatchNorm has an exactly zero gradient: both sides hold rounding noise."""
    return mode == "train" and k.endswith(".0.bias") and not k.startswith("out.")


def run(golden_dir, name, mode):
    g = np.load(os.path.join(golden_dir, name))
    n, ci, B, T = int(g["n_layers"]), int(g["channels_interval"]), int(g["B"]), int(g["T"])
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    noisy, clean = make_pair(B, T, int(g["pair_seed"]))
    return g, st, wa.mse_step(st, noisy, clean, n, ci, frozen_bn=(mode == "eval"))


@pytest.mark.parametrize("mode", ["train", "eval"])
def test_small_config_every_gradient_and_dx(golden_dir, mode):
    g, st, (loss, grads, stats, y, dx) = run(golden_dir, "autograd_small_n4_c8.npz", mode)
    assert abs(loss - float(g[f"{mode}:loss"])) <= REL * float(g[f"{mode}:loss"])
    assert rel_err(y, g[f"{mode}:y"]) <= REL
    assert dx.shape == g[f"{mode}:dx"].shape
    assert rel_err(dx, g[f"{mode}:dx"]) <= REL
    keys = [k[len(mode) + 6:] for k in g.files if k.startswith(f"{mode}:grad:")]
    assert sorted(keys) == sorted(grads) and len(keys) == 4 * (2 * 4 + 1) + 2
    worst = (0.0, "")
    for k in keys:
        want = g[f"{mode}:grad:{k}"]
        assert grads[k].shape == want.shape, k
        if noise_only(k, mode):
            assert np.abs(grads[k]).max() <= 1e-12 and np.abs(want).max() <= 1e-12, k
            continue
        worst = max(worst, (rel_err(grads[k], want), k))
    print(f"small {mode}: worst gradient rel err {worst[0]:.2e} ({worst[1]}), dx {rel_err(dx, g[f'{mode}:dx']):.2e}")
    assert worst[0] <= REL, worst
    for k, v in stats.items():
        assert rel_err(v, g[f"{mode}:stat:{k}"]) <= REL, k
        if mode == "eval":
            assert np.array_equal(g[f"{mode}:stat:{k}"], st[k]), k       # eval-mode BatchNorm leaves them untouched


@pytest.mark.parametrize("mode", ["train", "eval"])
def test_reference_architecture_short_frames(golden_dir, mode):
    g, st, (loss, grads, stats, y, dx) = run(golden_dir, "autograd_full_n12_c24_b2_t4096.npz", mode)
    assert abs(loss - float(g[f"{mode}:loss"])) <= REL * float(g[f"{mode}:loss"])
    assert rel_err(y, g[f"{mode}:y"]) <= REL
    for k, v in list(grads.items()) + [("x", dx)]:
        if noise_only(k, mode):
            continue
        norm = float(g[f"{mode}:gnorm:{k}"])
        assert abs(np.sqrt((v ** 2).sum()) - norm) <= REL * norm, k
        assert np.abs(v.reshape(-1)[g[f"{mode}:gidx:{k}"]] - g[f"{mode}:gval:{k}"]).max() <= REL * np.abs(v).max(), k
    for k, v in stats.items():
        assert rel_err(v, g[f"{mode}:stat:{k}"]) <= REL, k


@pytest.mark.parametrize("name,train_name", [("autograd_small_n4_c8.npz", "train_small_n4_c8.npz"),
                                             ("autograd_full_n12_c24_b2_t4096.npz", "train_full_n12_c24_b2_t4096.npz")])
def test_training_mode_matches_the_training_goldens(golden_dir, name, train_name):
    """Free cross-check of the two generators: the training-mode step with the input requiring grad is the training step."""
    g = np.load(os.path.join(golden_dir, name))
    t = np.load(os.path.join(golden_dir, train_name))
    for k in ("n_layers", "channels_interval", "B", "T", "state_seed", "pair_seed"):
        assert int(g[k]) == int(t[k]), k
    assert abs(float(g["train:loss"]) - float(t["loss"])) <= SAME * float(t["loss"])
    assert rel_err(g["train:y"], t["y"]) <= SAME
    pairs = [k for k in t.files if k.startswith(("grad:", "gnorm:", "gval:", "stat:"))]
    assert pairs
    for k in pairs:
        if noise_only(k.split(":", 1)[1], "train"):
            continue
        assert rel_err(g["train:" + k], t[k]) <= SAME, k
    for k in (k for k in t.files if k.startswith("gidx:")):
        assert np.array_equal(g["train:" + k], t[k]), k


def test_input_gradient_by_finite_differences():
    """Independent of the goldens: d loss / d x by central differences on a tiny network, both BatchNorm modes."""
    n, ci, B, T = 2, 8, 2, 16
    st = {k: v.astype(np.float64) for k, v in wo.make_state(n, ci, seed=5).items()}
    noisy, clean = make_pair(B, T, 7)
    noisy = noisy.astype(np.float64)
    rng = np.random.default_rng(4)
    for frozen in (False, True):
        _, grads, _, _, dx = wa.mse_step(st, noisy, clean, n, ci, frozen_bn=frozen)
        for fi in rng.integers(0, noisy.size, size=6):
            idx = np.unravel_index(fi, noisy.shape)
            h = 1e-6
            xp, xm = noisy.copy(), noisy.copy()
            xp[idx] += h
            xm[idx] -= h
            fd = (wa.mse_step(st, xp, clean, n, ci, frozen_bn=frozen)[0] - wa.mse_step(st, xm, clean, n, ci, frozen_bn=frozen)[0]) / (2 * h)
            assert abs(fd - dx[idx]) <= 1e-6 * max(1.0, abs(fd)) + 1e-9, (frozen, idx, fd, dx[idx])
        if frozen:                                          # and one parameter per kind through the frozen-statistics backward
            for key in ("encoder.0.main.0.bias", "encoder.1.main.1.weight", "decoder.1.main.0.weight"):
                idx = np.unravel_index(int(rng.integers(0, st[key].size)), st[key].shape)
                sp = {k: v.copy() for k, v in st.items()}
                sm = {k: v.copy() for k, v in st.items()}
                sp[key][idx] += 1e-6
                sm[key][idx] -= 1e-6
                fd = (wa.mse_step(sp, noisy, clean, n, ci, frozen_bn=True)[0] - wa.mse_step(sm, noisy, clean, n, ci, frozen_bn=True)[0]) / 2e-6
                assert abs(fd - grads[key][idx]) <= 1e-6 * max(1.0, abs(fd)) + 1e-9, (key, idx, fd, grads[key][idx])
