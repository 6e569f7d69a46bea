"""
oracle/gen_golden_autograd.py — generates tests/golden/autograd_*.npz by running autograd through the LIVE reference with an
input that requires grad, in training and in eval mode.

Run where a checkout of the reference exists (WUNET_REFERENCE, default /root/reference):

    python oracle/gen_golden_autograd.py

The unmodified ``model.unet_basic.Model`` (model/unet_basic.py:32) is cast to float64 and fed the seeded synthetic pair of
``gen_golden_train.py`` with ``x.requires_grad_(True)``; loss = ``nn.MSELoss()`` (model/loss.py:3-4), then ``backward()``.
Once in ``.train()`` mode (batch statistics; the same computation as tests/golden/train_*.npz, now with the input requiring
grad) and once in ``.eval()`` mode (BatchNorm normalises by the running statistics that ``make_state`` seeds: mean
0.1·randn, var U(0.5, 1.5)). Keys are prefixed "train:" / "eval:". Stored per mode: the loss, the output, the gradient of the
input and of every parameter (small config: in full; full config: norm and probes), and the running statistics after the
step. These vectors pin ``oracle/wunet_autograd_oracle.py`` (tests/test_autograd_oracle.py).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
REF = os.environ.get("WUNET_REFERENCE", "/root/reference")
sys.path.insert(0, REF)

from model.unet_basic import Model  # noqa: E402  (the unmodified reference)
from model.loss import mse_loss  # noqa: E402
from oracle import wunet_oracle as wo  # noqa: E402
from oracle.gen_golden_train import make_pair, probes  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def step(n, ci, state, noisy, clean, mode):
    m = Model(n_layers=n, channels_interval=ci)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in state.items()}, strict=True)
    m = m.double().train(mode == "train")
    x = torch.from_numpy(noisy).double().requires_grad_(True)
    y = m(x)
    loss = mse_loss()(torch.from_numpy(clean).double(), y)
    loss.backward()
    grads = {k: p.grad.detach().numpy() for k, p in m.named_parameters()}
    stats = {k: v.detach().numpy() for k, v in m.state_dict().items() if "running_" in k}
    return float(loss.detach()), y.detach().numpy(), x.grad.detach().numpy(), grads, stats


def main():
    torch.set_num_threads(os.cpu_count() or 1)
    os.makedirs(OUT, exist_ok=True)
    # ---- small config: every gradient stored ----------------------------------------------------------------
    n, ci, B, T = 4, 8, 3, 256
    st = wo.make_state(n, ci, seed=21)
    noisy, clean = make_pair(B, T, seed=22)
    out = dict(n_layers=n, channels_interval=ci, B=B, T=T, state_seed=21, pair_seed=22)
    for mode in ("train", "eval"):
        loss, y, dx, grads, stats = step(n, ci, st, noisy, clean, mode)
        out.update({f"{mode}:loss": loss, f"{mode}:y": y, f"{mode}:dx": dx})
        out.update({f"{mode}:grad:{k}": v for k, v in grads.items()})
        out.update({f"{mode}:stat:{k}": v for k, v in stats.items()})
    np.savez_compressed(os.path.join(OUT, "autograd_small_n4_c8.npz"), **out)
    # ---- reference architecture (12 x 24), short frames: norms + probes ----------------------------------------
    n, ci, B, T = 12, 24, 2, 4096
    st = wo.make_state(n, ci, seed=0)
    noisy, clean = make_pair(B, T, seed=23)
    out = dict(n_layers=n, channels_interval=ci, B=B, T=T, state_seed=0, pair_seed=23)
    for mode in ("train", "eval"):
        loss, y, dx, grads, stats = step(n, ci, st, noisy, clean, mode)
        out.update({f"{mode}:loss": loss, f"{mode}:y": y})
        for k, v in list(grads.items()) + [("x", dx)]:
            idx, val = probes(v)
            out[f"{mode}:gnorm:{k}"] = np.sqrt((v.astype(np.float64) ** 2).sum())
            out[f"{mode}:gidx:{k}"] = idx
            out[f"{mode}:gval:{k}"] = val
        out.update({f"{mode}:stat:{k}": v for k, v in stats.items()})
    np.savez_compressed(os.path.join(OUT, "autograd_full_n12_c24_b2_t4096.npz"), **out)
    print("wrote", sorted(f for f in os.listdir(OUT) if f.startswith("autograd_")))


if __name__ == "__main__":
    main()
