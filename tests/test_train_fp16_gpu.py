"""fp16 training step with in-library dz scaling, Model(train_precision="fp16_scaled") (DESIGN §5.4): the fp16 tensor-core
kernels pass by pass against float64 on the fp16-rounded, scaled operands, the whole step and the autograd goldens within the
tf32 tests' bars, the scaling's exactness (gradients of loss 2^m are 2^m times those of loss, bit for bit), non-finite values
reaching the gradients and a GradScaler, deterministic and SyncBatchNorm repeatability, and a 30-step Adam trajectory against
the fp32 native step."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_autograd_gpu as tag
import test_sync_bn_gpu as tsync
import test_train_bf16_gpu as tbf
import test_train_deterministic_gpu as tdet
import test_train_tf32_gpu as ttf
from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import _lib

pytestmark = [pytest.mark.gpu]

PREC = "fp16_scaled"
DIRECT, DECIM, UPCAT = tbf.DIRECT, tbf.DECIM, tbf.UPCAT
F16_ULP = 2.0 ** -10    # relative spacing of fp16 (10 explicit mantissa bits): bound of one round-to-nearest flip


def f16(a):
    """fp16 rounding (round to nearest even, overflow to inf) of fp32 values, as float64"""
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32))).half().double()


def scale_of(a):
    """2^k of the library's dz scaling for the values `a` (the host restatement of the kernels' rule)"""
    return 2.0 ** _lib.load().wunet_debug_train_dz_scale(float(np.abs(np.asarray(a, dtype=np.float32)).max()))


def run_pass(pss, mode, k, B, L, cin0, cin1, cout, src0, src1, w, dz):
    cin = cin0 + cin1
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    t = [dev(a) for a in (src0, src1, w, dz)]
    shape = {0: (B, cout, L), 1: (B, cin, L), 2: (cout, cin, k)}[pss]
    out = torch.empty(shape, dtype=torch.float32, device="cuda")
    ptr = lambda a: None if a is None else a.data_ptr()  # noqa: E731
    _lib.check(_lib.load().wunet_debug_train_conv(pss, _lib.PREC_FP16_SCALED, mode, k, B, L, cin0, cin1, cout,
                                                   *[ptr(a) for a in t], out.data_ptr()))
    return out.cpu().numpy().astype(np.float64)


@pytest.mark.parametrize("dz_scale", [1e-7, 1.0], ids=["dz1e-7", "dz1"])
@pytest.mark.parametrize("pss", [0, 1, 2], ids=["forward", "input_grad", "weight_grad"])
@pytest.mark.parametrize("shape", ttf.SHAPES, ids=[tbf._id(s) for s in ttf.SHAPES])
def test_debug_pass(shape, pss, dz_scale):
    """One pass through wunet_debug_train_conv at WUNET_PREC_FP16_SCALED against a float64 convolution of the fp16-rounded
    operands, dz rounded as fp16(dz 2^k) and the result multiplied by 2^-k, held to the tf32 test's bars (SUM_REL, WGRAD_REL
    of sum |products| per output; four fp16 flips per output where the kernel fuses the interpolation into one FMA). dz of
    about 1e-7, the size of the reference's upper-block gradients, would mostly flush to zero in fp16 without the scaling."""
    if pss == 0 and dz_scale != 1.0:
        pytest.skip("the forward reads no dz")
    k, mode, B, L, cin0, cin1, cout = shape
    if pss == 1 and mode != DIRECT:
        mode = DIRECT
        cin0, cin1 = cin0 + cin1, 0
    cin = cin0 + cin1
    pad = (k - 1) // 2
    g = np.random.default_rng(hash(shape) % 2**32 + 17 * pss + 7)
    src0 = g.standard_normal((B, cin0, {DIRECT: L, DECIM: 2 * L, UPCAT: L // 2}[mode])).astype(np.float32)
    src1 = g.standard_normal((B, cin1, L)).astype(np.float32) if mode == UPCAT else None
    w = (g.standard_normal((cout, cin, k)) / np.sqrt(cin * k)).astype(np.float32)
    dz = (dz_scale * g.standard_normal((B, cout, L))).astype(np.float32) if pss != 0 else None
    got = run_pass(pss, mode, k, B, L, cin0, cin1, cout, src0, src1, w, dz)

    xin = f16(tbf.block_input(mode, src0, src1, L)) if pss != 1 else None
    wr = f16(w)
    s = scale_of(dz) if dz is not None else 1.0
    dzr = f16(dz * np.float32(s)) if dz is not None else None
    if pss == 0:
        want = F.conv1d(xin, wr, padding=pad)
        mag = F.conv1d(xin.abs(), wr.abs(), padding=pad)
    elif pss == 1:
        want = F.conv_transpose1d(dzr, wr, padding=pad)
        mag = F.conv_transpose1d(dzr.abs(), wr.abs(), padding=pad)
    else:
        want = torch.nn.grad.conv1d_weight(xin, wr.shape, dzr, padding=pad)
        mag = torch.nn.grad.conv1d_weight(xin.abs(), wr.shape, dzr.abs(), padding=pad)
    want, mag = want.numpy() / s, mag.numpy() / s
    assert np.abs(want).max() > 0
    bar = (ttf.WGRAD_REL if pss == 2 else ttf.SUM_REL) * mag
    if mode == UPCAT and pss != 1:
        other = np.abs(w).max() if pss == 0 else np.abs(dz).max()
        bar = bar + 4 * F16_ULP * other * float(xin.abs().max())
    err = np.abs(got - want)
    worst = float((err / np.maximum(mag, 1e-300)).max())
    print(f"{tbf._id(shape)} pass {pss} fp16_scaled (dz ~ {dz_scale:g}, 2^k = {s:g}): worst |err| / sum|products| = {worst:.2e}")
    assert np.all(err <= bar), (worst, np.unravel_index(np.argmax(err - bar), err.shape))


@pytest.mark.parametrize("golden", sorted(tbf.FP32_BARS))
def test_step_vs_golden(golden_dir, golden, monkeypatch):
    """Native fp16_scaled against the float64 golden step, with the tf32 test's rule: loss, output, worst per-parameter
    gradient and running statistics each within max(2 x PyTorch-TF32's error, the fp32 native step's bar)."""
    g = np.load(f"{golden_dir}/{golden}")
    n, ci, B, T = int(g["n_layers"]), int(g["channels_interval"]), int(g["B"]), int(g["T"])
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    noisy, clean = tbf.make_pair(B, T, int(g["pair_seed"]))
    ttf.torch_tf32(monkeypatch)
    nat = tbf.step_errors(tbf.make_model(n, ci, st, "native", PREC), g, noisy, clean, autocast=False)
    tf = tbf.step_errors(tbf.make_model(n, ci, st, "native", "tf32"), g, noisy, clean, autocast=False)
    ref = tbf.step_errors(tbf.make_model(n, ci, st, "torch"), g, noisy, clean, autocast=False)
    names = ("loss rel", "y max-abs", "worst grad rel", "running stats rel")
    for name, a, b, c, bar in zip(names, nat, tf, ref, tbf.FP32_BARS[golden]):
        av, bv, cv = (a[0], b[0], c[0]) if isinstance(a, tuple) else (a, b, c)
        print(f"{golden} {name}: native fp16_scaled {av:.2e}{' (' + a[1] + ')' if isinstance(a, tuple) else ''}, "
              f"native tf32 {bv:.2e}, PyTorch TF32 {cv:.2e}, fp32 bar {bar:.0e}")
        assert av <= max(2 * cv, bar), (name, av, cv, bar)


@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("golden", [tag.SMALL, tag.FULL])
def test_autograd_goldens(golden_dir, golden, mode, monkeypatch):
    """x.grad in training mode and the eval-mode (frozen BatchNorm) step, same rule as above with test_autograd_gpu.py's
    bars; dx is held to the gradient bar."""
    g, n, ci, st, noisy, clean = tag.load(golden_dir, golden)
    ttf.torch_tf32(monkeypatch)
    nat = tag.step_errors(tag.make_model(n, ci, st, mode, "native", PREC), g, st, mode, noisy, clean)
    ref = tag.step_errors(tag.make_model(n, ci, st, mode, "torch"), g, st, mode, noisy, clean)
    loss_bar, y_bar, grad_bar = tag.FP32_BARS[(golden, mode)]
    names = ("loss rel", "y max-abs", "worst grad rel", "dx rel", "running stats rel")
    for name, a, c, bar in zip(names, nat, ref, (loss_bar, y_bar, grad_bar, grad_bar, 1e-5)):
        av, cv = (a[0], c[0]) if isinstance(a, tuple) else (a, c)
        print(f"{golden} {mode} {name}: native fp16_scaled {av:.2e}, PyTorch TF32 {cv:.2e}, bar {bar:.0e}")
        assert av <= max(2 * cv, bar), (name, av, cv, bar)


def _grads(st, n, ci, noisy, clean, m_exp, hook=None):
    """one deterministic step of loss 2^m_exp: the output, dx and every parameter gradient"""
    m = tag.make_model(n, ci, st, "train", train_precision=PREC)
    x = torch.from_numpy(noisy).cuda().requires_grad_(True)
    y = m(x)
    if hook is not None:
        y.register_hook(hook)
    (torch.nn.MSELoss()(torch.from_numpy(clean).cuda(), y) * 2.0 ** m_exp).backward()
    out = {"dx": x.grad}
    out.update({"grad:" + k: p.grad for k, p in m.named_parameters()})
    return out


@pytest.mark.parametrize("m_exp", [-24, 0, 16])
def test_scaling_is_exact(m_exp, monkeypatch):
    """Deterministic mode: every gradient of loss 2^m is 2^m times the gradient of loss, bit for bit. The per-block scale
    follows max |dz| by the same power of two, so the fp16 operands are the same bits. At m = -24 the upper blocks' dz (about
    1e-7 x 2^-24) lies below fp16's smallest subnormal: unscaled fp16 operands would be zero."""
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    n, ci, B, T = 12, 24, 2, 4096
    st = wo.make_state(n, ci, seed=31)
    noisy, clean = tag.make_pair(B, T, 32)
    base = _grads(st, n, ci, noisy, clean, 0)
    got = _grads(st, n, ci, noisy, clean, m_exp)
    for k, v in base.items():
        assert torch.isfinite(v).all(), k
        assert torch.equal(got[k], v * 2.0 ** m_exp), (k, float((got[k] - v * 2.0 ** m_exp).abs().max()))
    assert all(float(v.abs().max()) > 0 for k, v in got.items() if k.endswith(".weight")), "a weight gradient is zero"


def _poison(g):
    g = g.clone()
    g.view(-1)[g.numel() // 3] = float("inf")
    return g


def test_non_finite_dy_reaches_the_gradients():
    """An infinite entry of dy gives non-finite parameter gradients (fp16 stores do not saturate)."""
    n, ci, B, T = 4, 8, 3, 256
    st = wo.make_state(n, ci, seed=41)
    noisy, clean = tag.make_pair(B, T, 42)
    got = _grads(st, n, ci, noisy, clean, 0, hook=_poison)
    bad = [k for k, v in got.items() if not torch.isfinite(v).all()]
    assert "grad:out.0.weight" in bad and "dx" in bad, bad
    for part in ("decoder", "middle", "encoder"):                  # through every tensor-core block and down to block 0
        assert any(k.startswith("grad:" + part) for k in bad), (part, bad)


def test_grad_scaler_skips_a_non_finite_step():
    """torch.amp.GradScaler sees the non-finite gradients (found_inf) and skips the optimizer step: the parameters stay as
    they were; a finite step afterwards updates them."""
    n, ci, B, T = 4, 8, 3, 256
    st = wo.make_state(n, ci, seed=43)
    noisy, clean = tag.make_pair(B, T, 44)
    m = tag.make_model(n, ci, st, "train", train_precision=PREC)
    opt = torch.optim.SGD(m.parameters(), lr=1e-2)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 16)
    before = {k: p.detach().clone() for k, p in m.named_parameters()}
    y = m(torch.from_numpy(noisy).cuda())
    y.register_hook(_poison)
    scaler.scale(torch.nn.MSELoss()(torch.from_numpy(clean).cuda(), y)).backward()
    scaler.step(opt)
    scaler.update()
    assert scaler.get_scale() == 2.0 ** 15                    # the step was found non-finite and the scale backed off
    assert all(torch.equal(p, before[k]) for k, p in m.named_parameters())
    opt.zero_grad()
    scaler.scale(torch.nn.MSELoss()(torch.from_numpy(clean).cuda(), m(torch.from_numpy(noisy).cuda()))).backward()
    scaler.step(opt)
    scaler.update()
    assert all(torch.isfinite(p).all() for p in m.parameters())
    assert any(not torch.equal(p, before[k]) for k, p in m.named_parameters())


@pytest.mark.parametrize("case", [(4, 8, 3, 256), (12, 24, 2, 4096)], ids=["n4_c8", "n12_c24"])
def test_deterministic_step_is_bitwise_repeatable(case, monkeypatch):
    """torch.backends.cudnn.deterministic = True: two steps from the same state and batch give the same bits in the output,
    every parameter gradient, x.grad and the running buffers."""
    n, ci, B, T = case
    st = wo.make_state(n, ci, seed=21)
    noisy, clean = tag.make_pair(B, T, 22)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    runs = []
    for _ in range(2):
        m = tag.make_model(n, ci, st, "train", train_precision=PREC)
        x = torch.from_numpy(noisy).cuda().requires_grad_(True)
        y = m(x)
        torch.nn.MSELoss()(torch.from_numpy(clean).cuda(), y).backward()
        out = {"y": y.detach(), "dx": x.grad}
        out.update({"grad:" + k: p.grad for k, p in m.named_parameters()})
        out.update({k: v for k, v in m.state_dict().items() if "running_" in k})
        runs.append(out)
    assert torch.isfinite(runs[0]["y"]).all() and torch.isfinite(runs[0]["dx"]).all()
    tdet.assert_bitwise(runs[0], runs[1], "two deterministic fp16_scaled steps")


def test_syncbn_passthrough_reproduces_the_default_step(monkeypatch):
    """A pass-through SyncBatchNorm hook gives the bits of the step without one (each rank picks its own scales, so a
    single rank's step is unchanged by the hook)."""
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    n, ci, B, T = 12, 24, 3, 8192
    st = wo.make_state(n, ci, seed=11)
    noisy, clean = tsync.make_pair(B, T, 12)
    ref, _, _ = tsync.model_step(st, n, ci, PREC, noisy, clean, seam=False)
    got, n_fwd, n_bwd = tsync.model_step(st, n, ci, PREC, noisy, clean, seam=True)
    assert (n_fwd, n_bwd) == (2 * (2 * n + 1), 2 * n + 1)
    diff = [k for k in ref if not torch.equal(ref[k], got[k])]
    assert not diff, diff


def test_thirty_adam_steps_repeat_bit_for_bit(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    (la, sa), (lb, sb) = tdet.adam_run(PREC), tdet.adam_run(PREC)
    assert torch.isfinite(la).all()
    assert torch.equal(la, lb), (la - lb).abs().max()
    diff = [k for k in sa if not torch.equal(sa[k], sb[k])]
    assert not diff, diff[:10]


def test_adam_trajectory_tracks_fp32():
    """Reference architecture at T = 16384, one fixed batch of 4 frames, 30 Adam steps (lr 1e-3) from the same state, native
    fp16_scaled against native fp32: both losses fall, and the fp16_scaled loss stays within the tf32 test's band."""
    n, ci, B, T = 12, 24, 4, 16384
    st = wo.make_state(n, ci, seed=11)
    noisy, clean = tbf.make_pair(B, T, 123)
    curves = {}
    for prec in ("fp32", PREC):
        torch.manual_seed(0)
        m = tbf.make_model(n, ci, st, "native", prec)
        opt = torch.optim.Adam(m.parameters(), lr=1e-3, betas=(0.9, 0.999))
        losses = []
        for _ in range(30):
            opt.zero_grad()
            losses.append(tbf.step(m, noisy, clean)[0])
            opt.step()
        curves[prec] = np.array(losses)
    dev = np.abs(curves[PREC] - curves["fp32"]) / curves["fp32"]
    print("fp32 losses       ", np.array2string(curves["fp32"], precision=5))
    print("fp16_scaled losses", np.array2string(curves[PREC], precision=5))
    print(f"max relative deviation {dev.max():.3e} at step {int(dev.argmax())}")
    for prec, c in curves.items():
        assert c[-1] < c[0], (prec, c[0], c[-1])
    assert dev.max() <= ttf.TRAJ_BAND, dev


def test_scale_slots_hold_each_blocks_max_dz():
    """After a deterministic step on a workspace filled with NaN, the scale slot of every tensor-core block (layout field 22)
    holds max |dz| of that block, the value the kernels derive 2^k from (so the backward clears the slots itself), and dz
    is left unscaled in the workspace."""
    s = tdet.det_step("odd_lengths", PREC, "batch", True)
    tdet.det_run(s, tdet.fill_nan, want_dx=False)
    n, ci, B, T = s.n, s.ci, s.B, s.T
    for i in range(2 * n + 1):
        buf = (ctypes.c_longlong * 23)()
        _lib.check(_lib.load().wunet_debug_train_layout(n, ci, B, T, _lib.PREC_FP16_SCALED, i, buf, 23))
        if i == 0:
            assert buf[22] == -1                                 # block 0 stays fp32
            continue
        d = _lib.debug_train_layout(n, ci, B, T, i, PREC)
        dz = s.ws[d["ga"] // 4: d["ga"] // 4 + B * d["Cout"] * d["L"]]
        assert buf[22] > 0 and float(s.ws[buf[22] // 4]) == float(dz.abs().max()) > 0, i
