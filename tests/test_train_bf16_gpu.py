"""Mixed-precision training step, Model(train_precision="bf16") (DESIGN §5.4): the tensor-core kernels of wunet_train_tc.cu
at bf16 pass by pass, the whole step against the float64 golden steps next to PyTorch's own autocast step, and a
30-step Adam trajectory against the fp32 native step."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model, _lib

pytestmark = [pytest.mark.gpu]

DIRECT, DECIM, UPCAT = 0, 1, 2
SUM_REL = 1e-3        # per-output error bar, relative to sum |products| of that output (see test_debug_pass)
BF16_ULP = 2.0 ** -8  # relative spacing of bf16 (8 significant bits): bound of one round-to-nearest flip


def bf16(a):
    return torch.as_tensor(a).to(torch.bfloat16).to(torch.float64)


def upsample_f32(p, L):
    """F.interpolate(scale_factor=2, mode="linear", align_corners=True) with the fp32 index math of fetch_src."""
    Lin = p.shape[-1]
    scale = np.float32((Lin - 1) / (L - 1)) if L > 1 else np.float32(0)
    s = scale * np.arange(L, dtype=np.float32)
    i0 = s.astype(np.int64)
    i1 = np.where(i0 < Lin - 1, i0 + 1, i0)
    lam1 = (s - i0.astype(np.float32)).astype(np.float32)
    lam0 = (np.float32(1) - lam1).astype(np.float32)
    return (lam0 * p[..., i0] + lam1 * p[..., i1]).astype(np.float32)


def block_input(mode, src0, src1, L):
    if mode == DIRECT:
        return src0
    if mode == DECIM:
        return src0[..., ::2]
    return np.concatenate([upsample_f32(src0, L), src1], axis=1)


def run_pass(pss, prec, mode, k, B, L, cin0, cin1, cout, src0, src1, w, dz):
    cin = cin0 + cin1
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    t = [dev(a) for a in (src0, src1, w, dz)]
    shape = {0: (B, cout, L), 1: (B, cin, L), 2: (cout, cin, k)}[pss]
    out = torch.empty(shape, dtype=torch.float32, device="cuda")
    ptr = lambda a: None if a is None else a.data_ptr()  # noqa: E731
    _lib.check(_lib.load().wunet_debug_train_conv(pss, _lib.PRECISIONS[prec], mode, k, B, L, cin0, cin1, cout,
                                                   *[ptr(a) for a in t], out.data_ptr()))
    return out.cpu().numpy().astype(np.float64)


# (ksize, mode, B, L, Cin0, Cin1, Cout): every (ksize, mode) of the reference architecture and of the n4/c8 golden config;
# frames of 1 .. 8 samples (shorter than a tile), lengths that are not a multiple of the 128-row / 64-position tiles,
# B >= 3 (tiles next to frame edges), channel counts that are not multiples of 16 or 64, more than one 64-channel chunk
# and more than one 64-column tile
SHAPES = [
    (15, DECIM, 3, 1, 8, 0, 16),
    (15, DECIM, 3, 2, 16, 0, 24),
    (15, DECIM, 3, 4, 32, 0, 32),
    (15, DECIM, 3, 300, 24, 0, 32),
    (15, DECIM, 4, 130, 96, 0, 120),
    (15, DECIM, 3, 2048, 48, 0, 72),
    (15, DIRECT, 3, 200, 1, 0, 24),
    (15, DIRECT, 3, 8, 24, 0, 48),
    (5, UPCAT, 3, 2, 32, 32, 32),
    (5, UPCAT, 3, 8, 24, 32, 24),
    (5, UPCAT, 3, 300, 48, 24, 24),
    (5, UPCAT, 3, 256, 72, 48, 96),
    (5, UPCAT, 5, 4, 32, 24, 24),
]


def _id(s):
    return "k{}-{}-B{}-L{}-c{}+{}-o{}".format(s[0], ["direct", "decim", "upcat"][s[1]], *s[2:])


@pytest.mark.parametrize("prec", ["bf16", "fp32"])
@pytest.mark.parametrize("pss", [0, 1, 2], ids=["forward", "input_grad", "weight_grad"])
@pytest.mark.parametrize("shape", SHAPES, ids=[_id(s) for s in SHAPES])
def test_debug_pass(shape, pss, prec):
    """One pass through wunet_debug_train_conv against a float64 convolution of the operands the kernel multiplies: for
    "bf16" those are the bf16-rounded block input, weights and dz, which takes the rounding out of the comparison.

    Bar: |err| <= SUM_REL * sum_k |product_k| for every output. fp32 accumulation of n products is off by at most ~n * 2^-24
    of that sum (n <= 6144 here: 4e-4, typically far less). A wrong tap, channel offset, frame edge or swizzle moves an output
    by about its own size, ~ sum |products| / sqrt(n) for these random operands (>= 1e-2 of the sum), i.e. an order above the bar.
    Interpolated operands (mode UPCAT, forward and weight gradient) pass through fp32 arithmetic before the rounding; the
    kernel may fuse lam0 * a + lam1 * b into one FMA where numpy rounds twice, so a value a hair away from a bf16 rounding
    midpoint can round to the neighbouring bf16 value: one ulp (2^-8 relative) on that operand. Each such flip moves one
    product by at most 2^-8 * max|w| * max|x|; the bar allows four of them per output (a flip needs an fp32 result within an
    ulp of a midpoint, ~2^-16 of the values, so even one per output is rare)."""
    k, mode, B, L, cin0, cin1, cout = shape
    if pss == 1 and mode != DIRECT:
        mode = DIRECT                               # the input gradient reads dz as a plain [B][Cout][L] input
        cin0, cin1 = cin0 + cin1, 0
    cin = cin0 + cin1
    pad = (k - 1) // 2
    g = np.random.default_rng(hash(shape) % 2**32 + 17 * pss)
    src0 = g.standard_normal((B, cin0, {DIRECT: L, DECIM: 2 * L, UPCAT: L // 2}[mode])).astype(np.float32)
    src1 = g.standard_normal((B, cin1, L)).astype(np.float32) if mode == UPCAT else None
    w = (g.standard_normal((cout, cin, k)) / np.sqrt(cin * k)).astype(np.float32)
    dz = g.standard_normal((B, cout, L)).astype(np.float32) if pss != 0 else None
    got = run_pass(pss, prec, mode, k, B, L, cin0, cin1, cout, src0, src1, w, dz)

    rnd = bf16 if prec == "bf16" else (lambda a: torch.as_tensor(a).to(torch.float64))
    xin = rnd(block_input(mode, src0, src1, L)) if pss != 1 else None
    wr = rnd(w)
    dzr = rnd(dz) if dz is not None else None
    if pss == 0:
        want = F.conv1d(xin, wr, padding=pad)
        mag = F.conv1d(xin.abs(), wr.abs(), padding=pad)
    elif pss == 1:
        want = F.conv_transpose1d(dzr, wr, padding=pad)
        mag = F.conv_transpose1d(dzr.abs(), wr.abs(), padding=pad)
    else:
        want = torch.nn.grad.conv1d_weight(xin, wr.shape, dzr, padding=pad)
        mag = torch.nn.grad.conv1d_weight(xin.abs(), wr.shape, dzr.abs(), padding=pad)
    want, mag = want.numpy(), mag.numpy()
    bar = SUM_REL * mag
    if prec == "bf16" and mode == UPCAT and pss != 1:
        other = np.abs(w).max() if pss == 0 else np.abs(dz).max()
        bar = bar + 4 * BF16_ULP * other * float(xin.abs().max())
    err = np.abs(got - want)
    worst = float((err / np.maximum(mag, 1e-30)).max())
    print(f"{_id(shape)} pass {pss} {prec}: worst |err| / sum|products| = {worst:.2e}")
    assert np.all(err <= bar), (worst, np.unravel_index(np.argmax(err - bar), err.shape))


def make_pair(B, T, seed):
    g = np.random.Generator(np.random.PCG64(seed))
    clean = (0.1 * g.standard_normal((B, 1, T))).astype(np.float32)
    noisy = (clean + 0.05 * g.standard_normal((B, 1, T))).astype(np.float32)
    return noisy, clean


def make_model(n, ci, st, backend, train_precision="fp32"):
    m = Model(n, ci, precision="fp32", train_backend=backend, train_precision=train_precision)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    return m.to("cuda:0").train()


def step(m, noisy, clean, autocast=False):
    with torch.autocast("cuda", torch.bfloat16, enabled=autocast):
        y = m(torch.from_numpy(noisy).cuda())
        loss = torch.nn.MSELoss()(torch.from_numpy(clean).cuda(), y.float())      # trainer/trainer.py:36 argument order
    loss.backward()
    return float(loss.detach()), y.detach().float().cpu().numpy()


def rel_err(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


# the fp32 native step's bars in test_train_gpu.py: (loss relative, output max-abs, worst gradient relative, running stats)
FP32_BARS = {"train_small_n4_c8.npz": (1e-5, 1e-5, 2e-4, 1e-5), "train_full_n12_c24_b2_t4096.npz": (1e-4, 1e-3, 2e-2, 1e-5)}


def step_errors(m, g, noisy, clean, autocast):
    loss, y = step(m, noisy, clean, autocast)
    worst = (0.0, "")
    for k, p in m.named_parameters():
        if k.endswith(".0.bias") and not k.startswith("out."):
            continue                                # conv bias ahead of BatchNorm: its gradient is rounding noise
        got = p.grad.detach().cpu().numpy().astype(np.float64)
        if "grad:" + k in g.files:
            e = rel_err(got, g["grad:" + k])
        else:
            norm = float(g["gnorm:" + k])
            e1 = abs(np.sqrt((got ** 2).sum()) - norm) / norm
            e2 = np.abs(got.reshape(-1)[g["gidx:" + k]] - g["gval:" + k]).max() / np.abs(got).max()
            e = float(max(e1, e2))
        worst = max(worst, (e, k))
    sd = m.state_dict()
    stat = 0.0
    for k in [k[5:] for k in g.files if k.startswith("stat:")]:
        if "num_batches" in k:
            assert int(sd[k]) == 1, k
        else:
            stat = max(stat, rel_err(sd[k].cpu().numpy(), g["stat:" + k]))
    for k, v in sd.items():
        if k.endswith("num_batches_tracked"):
            assert int(v) == 1, k
    return abs(loss - float(g["loss"])) / float(g["loss"]), float(np.abs(y - g["y"]).max()), worst, stat


@pytest.mark.parametrize("golden", sorted(FP32_BARS))
def test_step_vs_golden_and_autocast(golden_dir, golden):
    """Native bf16 against the float64 golden step, next to PyTorch's own mixed-precision step (the composite path under
    torch.autocast(bfloat16), cuDNN) on the same state and batch: loss, output, worst per-parameter gradient and running
    statistics each within max(2 x autocast's error, the fp32 native step's bar)."""
    g = np.load(os.path.join(golden_dir, golden))
    n, ci, B, T = int(g["n_layers"]), int(g["channels_interval"]), int(g["B"]), int(g["T"])
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    noisy, clean = make_pair(B, T, int(g["pair_seed"]))
    nat = step_errors(make_model(n, ci, st, "native", "bf16"), g, noisy, clean, autocast=False)
    ac = step_errors(make_model(n, ci, st, "torch"), g, noisy, clean, autocast=True)
    bars = FP32_BARS[golden]
    names = ("loss rel", "y max-abs", "worst grad rel", "running stats rel")
    for name, a, b, bar in zip(names, nat, ac, bars):
        av, bv = (a[0], b[0]) if isinstance(a, tuple) else (a, b)
        print(f"{golden} {name}: native bf16 {av:.2e}{' (' + a[1] + ')' if isinstance(a, tuple) else ''}, "
              f"autocast {bv:.2e}{' (' + b[1] + ')' if isinstance(b, tuple) else ''}, fp32 bar {bar:.0e}")
        assert av <= max(2 * bv, bar), (name, av, bv, bar)


TRAJ_BAND = 0.15      # measured 7.1e-2 (largest at step 4) on an H100 80GB HBM3 at 700 W; about 2x margin


def test_adam_trajectory_bf16_tracks_fp32():
    """Reference architecture at T = 16384, one fixed batch of 4 frames, 30 Adam steps (lr 1e-3; train.py:31-35) from the same
    state, native bf16 against native fp32: both losses fall, and the bf16 loss stays within TRAJ_BAND (relative) of the fp32
    loss at every step. First measurement: both curves fall from 0.1275 to 0.0031-0.0032 in 30 steps, and the largest relative gap
    is 7.1e-2 (step 4) while the loss drops fastest; Adam turns the rounding differences of the gradients into slightly
    different steps, and the curves come back together (1-3e-2 over the last ten steps)."""
    n, ci, B, T = 12, 24, 4, 16384
    st = wo.make_state(n, ci, seed=11)
    noisy, clean = make_pair(B, T, 123)
    curves = {}
    for prec in ("fp32", "bf16"):
        torch.manual_seed(0)
        m = make_model(n, ci, st, "native", prec)
        opt = torch.optim.Adam(m.parameters(), lr=1e-3, betas=(0.9, 0.999))
        losses = []
        for _ in range(30):
            opt.zero_grad()
            losses.append(step(m, noisy, clean)[0])
            opt.step()
        curves[prec] = np.array(losses)
    dev = np.abs(curves["bf16"] - curves["fp32"]) / curves["fp32"]
    print("fp32 losses", np.array2string(curves["fp32"], precision=5))
    print("bf16 losses", np.array2string(curves["bf16"], precision=5))
    print(f"max relative deviation {dev.max():.3e} at step {int(dev.argmax())}")
    for prec, c in curves.items():
        assert c[-1] < c[0], (prec, c[0], c[-1])
    assert dev.max() <= TRAJ_BAND, dev
