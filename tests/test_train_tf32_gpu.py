"""TF32 training step, Model(train_precision="tf32") (DESIGN §5.4): the tensor-core kernels of wunet_train_tc.cu at tf32 pass by
pass against float64, the whole step and the autograd goldens next to PyTorch's own fp32 step with cuDNN's TF32 convolutions
(torch.backends.cudnn.allow_tf32, the reference's arithmetic on an H100), deterministic mode, and a 30-step Adam trajectory
against the fp32 native step."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_autograd_gpu as tag
import test_train_bf16_gpu as tbf
import test_train_blocks_gpu as tbl
import test_train_deterministic_gpu as tdet
from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model, _lib

pytestmark = [pytest.mark.gpu]

DIRECT, DECIM, UPCAT = tbf.DIRECT, tbf.DECIM, tbf.UPCAT
# Per-output error bars relative to sum |products|. Measured worst on an H100 80GB HBM3 at 700 W: 7.9e-7 (forward, input
# gradient) and 8.4e-6 (weight gradient, whose K = B L products per output is the longest fp32 accumulation of the three), so
# the weight gradient needs no wider bar than the other passes.
SUM_REL = 1e-4
WGRAD_REL = 1e-4
TF32_ULP = 2.0 ** -10   # relative spacing of tf32 (10 explicit mantissa bits): bound of one round-to-nearest flip

# SHAPES of the bf16 test, plus the reference's second encoder block at its training length (Cin 24 -> Cout 48, L = 8192)
SHAPES = tbf.SHAPES + [(15, DECIM, 2, 8192, 24, 0, 48)]


def tf32(a):
    """cvt.rna.tf32.f32 on the fp32 bits (round to nearest, ties away from zero: add half of the dropped 13 bits to the
    magnitude, then clear them), as float64"""
    u = np.ascontiguousarray(np.asarray(a, dtype=np.float32)).view(np.uint32)
    r = (u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)
    return torch.from_numpy(r.view(np.float32).astype(np.float64))


def test_tf32_emulation_is_round_to_nearest_ties_away():
    one = np.float32(1.0)
    half = np.float32(2.0 ** -11)               # half a tf32 ulp at 1
    got = tf32(np.array([1 + half, -(1 + half), 1 + half / 2, 1 + 1.5 * half], dtype=np.float32)).numpy()
    assert list(got) == [1 + 2 * half, -(1 + 2 * half), one, 1 + 2 * half]


def test_gpu_rounding_matches_the_emulation():
    """test_train_blocks_gpu.tf32r (the same rounding on int32 views of CUDA tensors, for the block check's tens of millions of
    operands) against tf32() above, bit for bit: ties and their neighbours in both signs, subnormals, the top of a binade
    (rounding up into the next one), the largest finite values (rounding up to infinity), zeros and random bit patterns."""
    pats = [0x3F801000, 0x3F800FFF, 0x3F801001, 0x3F803000, 0x3F802FFF,          # ties at 1 (odd and even kept bit), neighbours
            0x00000001, 0x00000FFF, 0x00001000, 0x00001FFF, 0x00003000, 0x007FF000, 0x007FFFFF,   # subnormals
            0x3FFFEFFF, 0x3FFFF000, 0x3FFFFFFF, 0x407FF000,                       # the top of a binade
            0x7F7FEFFF, 0x7F7FF000, 0x7F7FFFFF, 0x00000000, 0x00800000, 0x3DCCCCCD]
    rng = np.random.default_rng(3)
    exps = rng.integers(0, 255, 4096, dtype=np.uint32) << np.uint32(23)      # finite exponents, including subnormals
    bits = np.concatenate([np.array(pats, dtype=np.uint32), exps | rng.integers(0, 1 << 23, 4096, dtype=np.uint32)])
    bits = np.concatenate([bits, bits | np.uint32(0x80000000)])
    vals = bits.view(np.float32)
    want = tf32(vals).numpy().astype(np.float32).view(np.uint32)
    got = tbl.tf32r(torch.from_numpy(vals).cuda()).float().cpu().numpy().view(np.uint32)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(hex(bits[i]), hex(got[i]), hex(want[i])) for i in bad[:10]]
    assert want[0] == 0x3F802000 and want[1] == 0x3F800000 and want[18] == 0x7F800000     # ties away; top rounds to inf


def run_pass(pss, mode, k, B, L, cin0, cin1, cout, src0, src1, w, dz):
    cin = cin0 + cin1
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    t = [dev(a) for a in (src0, src1, w, dz)]
    shape = {0: (B, cout, L), 1: (B, cin, L), 2: (cout, cin, k)}[pss]
    out = torch.empty(shape, dtype=torch.float32, device="cuda")
    ptr = lambda a: None if a is None else a.data_ptr()  # noqa: E731
    _lib.check(_lib.load().wunet_debug_train_conv(pss, _lib.PREC_TF32, mode, k, B, L, cin0, cin1, cout,
                                                   *[ptr(a) for a in t], out.data_ptr()))
    return out.cpu().numpy().astype(np.float64)


@pytest.mark.parametrize("pss", [0, 1, 2], ids=["forward", "input_grad", "weight_grad"])
@pytest.mark.parametrize("shape", SHAPES, ids=[tbf._id(s) for s in SHAPES])
def test_debug_pass(shape, pss):
    """One pass through wunet_debug_train_conv at WUNET_PREC_TF32 against a float64 convolution of the tf32-rounded operands
    (the rounding emulated bit for bit above), which takes the rounding out of the comparison. What is left is fp32
    accumulation, held to SUM_REL (WGRAD_REL for the weight gradient) of sum |products| per output; a wrong tap, channel,
    frame edge or swizzle moves an output by ~ sum |products| / sqrt(n) (>= 1e-2 of the sum here). Interpolated operands
    (UPCAT, forward and weight gradient) may round to the neighbouring tf32 value where the kernel fuses the interpolation into
    one FMA and numpy does not: four such flips per output are allowed, as in the bf16 test."""
    k, mode, B, L, cin0, cin1, cout = shape
    if pss == 1 and mode != DIRECT:
        mode = DIRECT                               # the input gradient reads dz as a plain [B][Cout][L] input
        cin0, cin1 = cin0 + cin1, 0
    cin = cin0 + cin1
    pad = (k - 1) // 2
    g = np.random.default_rng(hash(shape) % 2**32 + 17 * pss + 5)
    src0 = g.standard_normal((B, cin0, {DIRECT: L, DECIM: 2 * L, UPCAT: L // 2}[mode])).astype(np.float32)
    src1 = g.standard_normal((B, cin1, L)).astype(np.float32) if mode == UPCAT else None
    w = (g.standard_normal((cout, cin, k)) / np.sqrt(cin * k)).astype(np.float32)
    dz = g.standard_normal((B, cout, L)).astype(np.float32) if pss != 0 else None
    got = run_pass(pss, mode, k, B, L, cin0, cin1, cout, src0, src1, w, dz)

    xin = tf32(tbf.block_input(mode, src0, src1, L)) if pss != 1 else None
    wr = tf32(w)
    dzr = tf32(dz) if dz is not None else None
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
    bar = (WGRAD_REL if pss == 2 else SUM_REL) * mag
    if mode == UPCAT and pss != 1:
        other = np.abs(w).max() if pss == 0 else np.abs(dz).max()
        bar = bar + 4 * TF32_ULP * other * float(xin.abs().max())
    err = np.abs(got - want)
    worst = float((err / np.maximum(mag, 1e-30)).max())
    print(f"{tbf._id(shape)} pass {pss} tf32: worst |err| / sum|products| = {worst:.2e}")
    assert np.all(err <= bar), (worst, np.unravel_index(np.argmax(err - bar), err.shape))


def torch_tf32(monkeypatch):
    """PyTorch's fp32 step with cuDNN's TF32 convolutions (its default on an H100)"""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", True)


@pytest.mark.parametrize("golden", sorted(tbf.FP32_BARS))
def test_step_vs_golden_and_torch_tf32(golden_dir, golden, monkeypatch):
    """Native tf32 against the float64 golden step, next to PyTorch's composite fp32 step with cuDNN TF32 on the same state
    and batch: loss, output, worst per-parameter gradient and running statistics each within max(2 x PyTorch-TF32's error,
    the fp32 native step's bar). The native bf16 step's errors are printed beside them."""
    g = np.load(f"{golden_dir}/{golden}")
    n, ci, B, T = int(g["n_layers"]), int(g["channels_interval"]), int(g["B"]), int(g["T"])
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    noisy, clean = tbf.make_pair(B, T, int(g["pair_seed"]))
    torch_tf32(monkeypatch)
    nat = tbf.step_errors(tbf.make_model(n, ci, st, "native", "tf32"), g, noisy, clean, autocast=False)
    bf16 = tbf.step_errors(tbf.make_model(n, ci, st, "native", "bf16"), g, noisy, clean, autocast=False)
    ref = tbf.step_errors(tbf.make_model(n, ci, st, "torch"), g, noisy, clean, autocast=False)
    names = ("loss rel", "y max-abs", "worst grad rel", "running stats rel")
    for name, a, b, c, bar in zip(names, nat, bf16, ref, tbf.FP32_BARS[golden]):
        av, bv, cv = (a[0], b[0], c[0]) if isinstance(a, tuple) else (a, b, c)
        print(f"{golden} {name}: native tf32 {av:.2e}{' (' + a[1] + ')' if isinstance(a, tuple) else ''}, native bf16 {bv:.2e}, "
              f"PyTorch TF32 {cv:.2e}, fp32 bar {bar:.0e}")
        assert av <= max(2 * cv, bar), (name, av, cv, bar)


@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("golden", [tag.SMALL, tag.FULL])
def test_autograd_goldens(golden_dir, golden, mode, monkeypatch):
    """x.grad in training mode and the eval-mode (frozen BatchNorm) step at tf32, same rule as above with
    test_autograd_gpu.py's bars; dx is held to the gradient bar."""
    g, n, ci, st, noisy, clean = tag.load(golden_dir, golden)
    torch_tf32(monkeypatch)
    nat = tag.step_errors(tag.make_model(n, ci, st, mode, "native", "tf32"), g, st, mode, noisy, clean)
    bf16 = tag.step_errors(tag.make_model(n, ci, st, mode, "native", "bf16"), g, st, mode, noisy, clean)
    ref = tag.step_errors(tag.make_model(n, ci, st, mode, "torch"), g, st, mode, noisy, clean)
    loss_bar, y_bar, grad_bar = tag.FP32_BARS[(golden, mode)]
    names = ("loss rel", "y max-abs", "worst grad rel", "dx rel", "running stats rel")
    for name, a, b, c, bar in zip(names, nat, bf16, ref, (loss_bar, y_bar, grad_bar, grad_bar, 1e-5)):
        av, bv, cv = (a[0], b[0], c[0]) if isinstance(a, tuple) else (a, b, c)
        print(f"{golden} {mode} {name}: native tf32 {av:.2e}, native bf16 {bv:.2e}, PyTorch TF32 {cv:.2e}, bar {bar:.0e}")
        assert av <= max(2 * cv, bar), (name, av, cv, bar)


@pytest.mark.parametrize("mode", ["train", "eval"])
def test_frozen_model_gets_the_same_input_gradient(mode):
    """requires_grad_(False) on every parameter: the dx-only backward gives the bits of the full backward's dx."""
    n, ci, B, T = 12, 24, 2, 4096
    st = wo.make_state(n, ci, seed=4)
    noisy, clean = tag.make_pair(B, T, 10)
    _, y_full, dx_full = tag.step(tag.make_model(n, ci, st, mode, train_precision="tf32"), noisy, clean)
    frozen = tag.make_model(n, ci, st, mode, train_precision="tf32").requires_grad_(False)
    _, y, dx = tag.step(frozen, noisy, clean)
    assert np.array_equal(y, y_full)
    assert np.array_equal(dx, dx_full)
    assert all(p.grad is None for p in frozen.parameters())


@pytest.mark.parametrize("case", [(4, 8, 3, 256), (12, 24, 2, 4096)], ids=["n4_c8", "n12_c24"])
def test_deterministic_step_is_bitwise_repeatable(case, monkeypatch):
    """torch.backends.cudnn.deterministic = True: two tf32 steps from the same state and batch give the same bits in the
    output, every parameter gradient, x.grad and the running buffers."""
    n, ci, B, T = case
    st = wo.make_state(n, ci, seed=21)
    noisy, clean = tag.make_pair(B, T, 22)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    runs = []
    for _ in range(2):
        m = tag.make_model(n, ci, st, "train", train_precision="tf32")
        x = torch.from_numpy(noisy).cuda().requires_grad_(True)
        y = m(x)
        torch.nn.MSELoss()(torch.from_numpy(clean).cuda(), y).backward()
        out = {"y": y.detach(), "dx": x.grad}
        out.update({"grad:" + k: p.grad for k, p in m.named_parameters()})
        out.update({k: v for k, v in m.state_dict().items() if "running_" in k})
        runs.append(out)
    assert torch.isfinite(runs[0]["y"]).all() and torch.isfinite(runs[0]["dx"]).all()
    tdet.assert_bitwise(runs[0], runs[1], "two deterministic tf32 steps")


@pytest.mark.parametrize("switch", ["cudnn", "algorithms"])
def test_thirty_adam_steps_repeat_bit_for_bit(switch, monkeypatch):
    if switch == "cudnn":
        monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    else:
        saved = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(True)
    try:
        (la, sa), (lb, sb) = tdet.adam_run("tf32"), tdet.adam_run("tf32")
    finally:
        if switch != "cudnn":
            torch.use_deterministic_algorithms(saved)
    assert torch.isfinite(la).all()
    assert torch.equal(la, lb), (la - lb).abs().max()
    diff = [k for k in sa if not torch.equal(sa[k], sb[k])]
    assert not diff, diff[:10]


TRAJ_BAND = 0.07      # measured 3.5e-2 (largest at step 12) on an H100 80GB HBM3 at 700 W; about 2x margin (bf16's: 0.15)


def test_adam_trajectory_tf32_tracks_fp32():
    """Reference architecture at T = 16384, one fixed batch of 4 frames, 30 Adam steps (lr 1e-3) from the same state, native
    tf32 against native fp32: both losses fall, and the tf32 loss stays within TRAJ_BAND (relative) of the fp32 loss."""
    n, ci, B, T = 12, 24, 4, 16384
    st = wo.make_state(n, ci, seed=11)
    noisy, clean = tbf.make_pair(B, T, 123)
    curves = {}
    for prec in ("fp32", "tf32"):
        torch.manual_seed(0)
        m = tbf.make_model(n, ci, st, "native", prec)
        opt = torch.optim.Adam(m.parameters(), lr=1e-3, betas=(0.9, 0.999))
        losses = []
        for _ in range(30):
            opt.zero_grad()
            losses.append(tbf.step(m, noisy, clean)[0])
            opt.step()
        curves[prec] = np.array(losses)
    dev = np.abs(curves["tf32"] - curves["fp32"]) / curves["fp32"]
    print("fp32 losses", np.array2string(curves["fp32"], precision=5))
    print("tf32 losses", np.array2string(curves["tf32"], precision=5))
    print(f"max relative deviation {dev.max():.3e} at step {int(dev.argmax())}")
    for prec, c in curves.items():
        assert c[-1] < c[0], (prec, c[0], c[-1])
    assert dev.max() <= TRAJ_BAND, dev


def test_c_abi_accepts_tf32_for_training_only():
    """The training entry points take WUNET_PREC_TF32 (with and without deterministic mode); every inference entry point
    refuses it with WUNET_EINVAL."""
    lib = _lib.load()
    m = Model(4, 8)
    c = m._context(torch.device("cuda:0"))
    try:
        B, T = 2, 256
        base = lib.wunet_train_workspace_bytes_prec(c, B, T, _lib.PREC_TF32)
        assert base > lib.wunet_train_workspace_bytes_prec(c, B, T, _lib.PREC_FP32) > 0
        assert lib.wunet_train_workspace_bytes_ex(c, B, T, _lib.PREC_TF32, 0) == base
        assert lib.wunet_train_workspace_bytes_ex(c, B, T, _lib.PREC_TF32, _lib.TRAIN_DETERMINISTIC) > base
        assert lib.wunet_workspace_bytes(c, B, T, _lib.PREC_TF32) == 0
        x = torch.zeros(B, 1, T, device="cuda")
        y = torch.empty_like(x)
        ws = torch.empty(1 << 24, dtype=torch.uint8, device="cuda")
        m = m.cuda().eval()
        with torch.no_grad():
            m(x)                                             # weights set, so only the precision can be wrong below
        EINVAL = -1
        assert lib.wunet_forward(c, x.data_ptr(), y.data_ptr(), B, T, _lib.PREC_TF32, ws.data_ptr(), ws.numel(), None) == EINVAL
        xh, yh = torch.zeros(B, 1, T), torch.empty(B, 1, T)
        assert lib.wunet_forward_host(c, xh.data_ptr(), yh.data_ptr(), B, T, _lib.PREC_TF32) == EINVAL
        ticket = ctypes.c_int(0)
        assert lib.wunet_stream_submit(c, xh.data_ptr(), yh.data_ptr(), B, T, _lib.PREC_TF32, ctypes.byref(ticket)) == EINVAL
        out = torch.empty(B, 8, T, device="cuda")
        assert lib.wunet_read_level(c, 0, ws.data_ptr(), B, T, _lib.PREC_TF32, out.data_ptr(), None) == EINVAL
        torch.cuda.synchronize()
    finally:
        m._release()
