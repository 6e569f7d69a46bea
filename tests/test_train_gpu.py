"""Native training step (SURVEY §8f row N1; wunet_train_forward / wunet_train_backward through Model(train_backend="native"))
against the training oracle's golden vectors and the composite PyTorch path.

Tolerances: the train-mode forward of the fp32 reference module itself differs from its float64 evaluation by 3.5-4.6e-4
(SURVEY §8c noise floors: batch-statistics BatchNorm amplifies rounding), so the forward is held to Y_TOL = 1e-3 of the
float64 golden output and the loss to 1e-4 relative; gradients to GRAD_REL of the largest entry (measured <= 2e-4 on the
small configuration)."""
import os

import numpy as np
import pytest
import torch

from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model

pytestmark = [pytest.mark.gpu]

GRAD_REL = 2e-4       # fp32 kernels vs the float64 reference step; relative to the largest entry of each gradient
GRAD_REL_FULL = 2e-2  # 25 blocks deep, batch statistics over 2 x L samples only: the reference's OWN fp32 autograd (PyTorch CPU)
                      # is 9.98e-3 away from the float64 golden step on decoder.6 BatchNorm.weight (measured), ours 9.2e-3
Y_TOL = 1e-3          # train-mode forward vs the float64 golden output (see the module docstring)


def make_pair(B, T, seed):
    g = np.random.Generator(np.random.PCG64(seed))
    clean = (0.1 * g.standard_normal((B, 1, T))).astype(np.float32)
    noisy = (clean + 0.05 * g.standard_normal((B, 1, T))).astype(np.float32)
    return noisy, clean


def make_model(n, ci, st, backend):
    m = Model(n, ci, precision="fp32", train_backend=backend)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    return m.to("cuda:0").train()


def step(m, noisy, clean):
    y = m(torch.from_numpy(noisy).cuda())
    loss = torch.nn.MSELoss()(torch.from_numpy(clean).cuda(), y)          # trainer/trainer.py:36 argument order
    loss.backward()
    return float(loss.detach()), y.detach().cpu().numpy()


def rel_err(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def test_small_config_step_vs_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "train_small_n4_c8.npz"))
    n, ci, B, T = int(g["n_layers"]), int(g["channels_interval"]), int(g["B"]), int(g["T"])
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    noisy, clean = make_pair(B, T, int(g["pair_seed"]))
    m = make_model(n, ci, st, "native")
    loss, y = step(m, noisy, clean)
    assert abs(loss - float(g["loss"])) <= 1e-5 * float(g["loss"])
    assert np.abs(y - g["y"]).max() <= 1e-5
    for k, p in m.named_parameters():
        want = g["grad:" + k]
        got = p.grad.cpu().numpy()
        if k.endswith(".0.bias") and not k.startswith("out."):
            assert np.abs(got).max() <= 1e-5 * max(np.abs(g["grad:" + k.replace(".0.bias", ".0.weight")]).max(), 1e-30), k
            continue
        assert rel_err(got, want) <= GRAD_REL, k
    sd = m.state_dict()
    for k in [k[5:] for k in g.files if k.startswith("stat:")]:
        if "num_batches" in k:
            assert int(sd[k]) == 1
        else:
            assert rel_err(sd[k].cpu().numpy(), g["stat:" + k]) <= 1e-5, k


def test_reference_architecture_step_vs_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "train_full_n12_c24_b2_t4096.npz"))
    n, ci, B, T = int(g["n_layers"]), int(g["channels_interval"]), int(g["B"]), int(g["T"])
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    noisy, clean = make_pair(B, T, int(g["pair_seed"]))
    m = make_model(n, ci, st, "native")
    loss, y = step(m, noisy, clean)
    yerr = float(np.abs(y - g["y"]).max())
    worst = (0.0, "")
    for k, p in m.named_parameters():
        if k.endswith(".0.bias") and not k.startswith("out."):
            continue
        got = p.grad.cpu().numpy().astype(np.float64)
        norm = float(g["gnorm:" + k])
        e1 = abs(np.sqrt((got ** 2).sum()) - norm) / norm
        e2 = np.abs(got.reshape(-1)[g["gidx:" + k]] - g["gval:" + k]).max() / np.abs(got).max()
        worst = max(worst, (float(max(e1, e2)), k))
    print(f"full architecture train step: loss rel err {abs(loss - float(g['loss'])) / float(g['loss']):.2e}, "
          f"y max-abs err {yerr:.2e}, worst gradient rel err {worst[0]:.2e} ({worst[1]})")
    assert abs(loss - float(g["loss"])) <= 1e-4 * float(g["loss"])
    assert yerr <= Y_TOL
    assert worst[0] <= GRAD_REL_FULL, worst


def test_three_adam_steps_track_the_composite_torch_path(monkeypatch):
    """trainer/trainer.py:34-38 + train.py:31-35 (Adam lr 1e-3): the same three steps on both backends stay together."""
    # both sides in true fp32: cuDNN's default TF32 convolutions (10-bit mantissa) would put the composite path's own
    # rounding far above the native path's
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    n, ci, B, T = 4, 8, 4, 256
    st = wo.make_state(n, ci, seed=31)
    ms = [make_model(n, ci, st, b) for b in ("native", "torch")]
    opts = [torch.optim.Adam(m.parameters(), lr=1e-3, betas=(0.9, 0.999)) for m in ms]
    for it in range(3):
        noisy, clean = make_pair(B, T, 40 + it)
        losses = []
        for m, opt in zip(ms, opts):
            opt.zero_grad()
            losses.append(step(m, noisy, clean)[0])
            opt.step()
        # after the first update the two trajectories differ by Adam's +-lr steps on rounding-noise gradients
        assert abs(losses[0] - losses[1]) <= (1e-4 if it == 0 else 2e-3) * abs(losses[1]), (it, losses)
    for (k, a), (_, b) in zip(ms[0].state_dict().items(), ms[1].state_dict().items()):
        if k.endswith(".0.bias") and not k.startswith("out."):
            continue                      # gradient is rounding noise, Adam turns it into +-lr steps on both sides
        # Adam normalises the update: where a gradient entry is rounding noise its sign (hence a full +-lr step per iteration)
        # differs between the backends, so parameters may sit 3 steps x 2 lr apart; relative to max |w| ~ 0.2 that is 3e-2
        assert np.abs(a.float().cpu().numpy() - b.float().cpu().numpy()).max() <= 3 * 2 * 1e-3 * 1.05, k


def test_tuned_training_kernels_match_the_one_thread_per_output_ones(monkeypatch):
    """csrc/wunet_train.cu: forward conv / input gradient through the tuned fp32 conv kernels and the tiled weight-gradient
    kernel against the naive kernels they replaced (WUNET_TRAIN_NAIVE=1), same step, reference architecture at T=4096."""
    n, ci, B, T = 12, 24, 3, 4096
    st = wo.make_state(n, ci, seed=5)
    noisy, clean = make_pair(B, T, 77)
    out = {}
    for naive in ("1", "0"):
        monkeypatch.setenv("WUNET_TRAIN_NAIVE", naive)
        m = make_model(n, ci, st, "native")
        loss, y = step(m, noisy, clean)
        out[naive] = (loss, y, {k: p.grad.detach().cpu().numpy() for k, p in m.named_parameters()},
                      {k: v.detach().cpu().numpy() for k, v in m.state_dict().items() if "running" in k})
    assert abs(out["0"][0] - out["1"][0]) <= 1e-6 * abs(out["1"][0])
    assert np.abs(out["0"][1] - out["1"][1]).max() <= 1e-5
    worst = (0.0, "")
    for k, g1 in out["1"][2].items():
        if k.endswith(".0.bias") and not k.startswith("out."):
            continue
        worst = max(worst, (rel_err(out["0"][2][k], g1), k))
    print(f"tuned vs naive training kernels: worst gradient rel diff {worst[0]:.2e} ({worst[1]})")
    assert worst[0] <= 2e-3, worst               # different summation orders of an ill-conditioned fp32 sum (see GRAD_REL_FULL)
    for k, v in out["1"][3].items():
        assert rel_err(out["0"][3][k], v) <= 1e-5, k
