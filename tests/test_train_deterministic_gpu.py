"""Deterministic mode of the native training step (WUNET_TRAIN_DETERMINISTIC; torch.backends.cudnn.deterministic or
torch.use_deterministic_algorithms in Python): the step must give the same bits every time, and stay as accurate as the
default step.

Repeatability: the C ABI runs on workspaces this test owns, pre-filled differently (zeros, NaN bytes, random bytes), so a
read of workspace memory the step did not write would show. y, the running buffers, every parameter gradient and dx must be
bitwise equal over three runs, and the backward split into part 0 and part 1 (data-parallel overlap) must equal the whole one.

Accuracy, restated from the default step's tests: fp32 against the float64 golden steps at (loss relative, y max-abs, worst
gradient relative to its largest entry, running statistics relative) = (1e-5, 1e-5, 2e-4, 1e-5) for train_small_n4_c8 and
(1e-4, 1e-3, 2e-2, 1e-5) for train_full_n12_c24_b2_t4096; bf16 within max(2 x the error of PyTorch's autocast step, that
fp32 bar). The autograd goldens keep test_autograd_gpu.py's bars. Block by block, each deterministic weight gradient is held
to WGRAD_REL and each head gradient to HEAD_REL of sum |products| against float64 (test_train_blocks_gpu.py's bars)."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

import test_autograd_gpu as tag
import test_train_bf16_gpu as tbf
import test_train_blocks_gpu as tbl
from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model, _lib

pytestmark = [pytest.mark.gpu]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DET = _lib.TRAIN_DETERMINISTIC
TRAIN_BARS = {"train_small_n4_c8.npz": (1e-5, 1e-5, 2e-4, 1e-5), "train_full_n12_c24_b2_t4096.npz": (1e-4, 1e-3, 2e-2, 1e-5)}
AUTOGRAD_BARS = {(tag.SMALL, "train"): (1e-5, 1e-5, 2e-4), (tag.FULL, "train"): (1e-4, 1e-3, 2e-2),
                 (tag.SMALL, "eval"): (1e-5, 1e-4, 2e-4), (tag.FULL, "eval"): (1e-5, 1e-4, 2e-5)}
assert tbl.WGRAD_REL == {"fp32": 1e-5, "bf16": 1e-3, "tf32": 3e-4, "fp16_scaled": 1e-3} and tbl.HEAD_REL == 1e-4


def fill_zeros(ws):
    ws.zero_()


def fill_nan(ws):
    ws.fill_(0xFF)                                       # every float reads as NaN


def fill_random(ws):
    ws.random_(0, 256, generator=torch.Generator(device=ws.device).manual_seed(1234))


def det_step(case, prec, mode, pgrads):
    s = tbl.Step(case, prec, mode, pgrads)              # its default-mode forward gives dy; the runs below redo the step
    s.flags |= DET
    return s


def det_run(s, fill, want_dx, split=False):
    """One deterministic step of `s` from its initial state on a fresh workspace filled by `fill` -> every output."""
    for v, v0 in zip(s.rm + s.rv, s.rm0 + s.rv0):
        v.copy_(v0)
    nbytes = s.lib.wunet_train_workspace_bytes_ex(s.ctx, s.B, s.T, _lib.TRAIN_PRECISIONS[s.prec], s.flags)
    assert nbytes > 0
    s.ws = None
    ws = torch.empty(nbytes, dtype=torch.uint8, device=s.dev)
    fill(ws)
    s.ws = ws.view(torch.float32)
    s.y.fill_(float("nan"))
    _lib.check(s.forward_rc())
    G = s.new_grads()
    dx = torch.full_like(s.x, float("nan")) if want_dx else None
    if split:
        s.backward(s.ws, G, None, 0)
        s.backward(s.ws, G, dx, 1)
    else:
        s.backward(s.ws, G, dx, -1)
    torch.cuda.synchronize()
    out = {"y": s.y.clone()}
    out.update({f"running_mean.{i}": v.clone() for i, v in enumerate(s.rm)})
    out.update({f"running_var.{i}": v.clone() for i, v in enumerate(s.rv)})
    if G is not None:
        for k in ("w", "b", "gamma", "beta"):
            out.update({f"{k}.{i}": v for i, v in enumerate(G[k])})
        out["wo"], out["bo"] = G["wo"], G["bo"]
    if dx is not None:
        out["dx"] = dx
    return out, G, dx


def assert_bitwise(a, b, what):
    assert a.keys() == b.keys()
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, f"{what}: not bit-identical: {diff[:10]}"


# (case of test_train_blocks_gpu.CASES, precision, BatchNorm mode, parameter gradients, dx)
REPEAT = ([("production", p, "batch", True, True) for p in ("fp32", "bf16", "tf32")] +
          [("odd_lengths", p, m, True, dx) for p in ("fp32", "bf16", "tf32") for m in ("batch", "frozen") for dx in (True, False)] +
          [("channel_plan", p, "batch", True, True) for p in ("fp32", "bf16")] +
          [("odd_lengths", p, "frozen", False, True) for p in ("fp32", "bf16", "tf32")])


def _rid(r):
    c, p, m, g, dx = r
    return f"{c}-{p}-{m}" + ("" if g else "-no_param_grads") + ("-dx" if dx else "")


@pytest.mark.parametrize("run", REPEAT, ids=[_rid(r) for r in REPEAT])
def test_step_is_bitwise_repeatable(run):
    case, prec, mode, pgrads, want_dx = run
    s = det_step(case, prec, mode, pgrads)
    try:
        outs = [det_run(s, f, want_dx)[0] for f in (fill_zeros, fill_nan, fill_random)]
        for f in ("y", "dx", "w.0", "wo"):
            if f in outs[0]:
                assert torch.isfinite(outs[0][f]).all(), f
        assert_bitwise(outs[0], outs[1], "zeros vs NaN workspace")
        assert_bitwise(outs[0], outs[2], "zeros vs random workspace")
        split = det_run(s, fill_nan, want_dx, split=True)[0]
        assert_bitwise(outs[0], split, "part -1 vs part 0 + part 1")
    finally:
        s.ws = None
        s.lib.wunet_destroy(s.ctx)


@pytest.mark.parametrize("run", [(c, p) for c in ("production", "channel_plan") for p in ("fp32", "bf16", "tf32")],
                         ids=lambda r: f"{r[0]}-{r[1]}")
def test_deterministic_gradients_block_by_block(run):
    """The whole deterministic step against float64 recomputed from its own workspace, block by block, at the block test's
    bars: the weight gradients at WGRAD_REL, the head gradients at HEAD_REL of sum |products|."""
    case, prec = run
    s = det_step(case, prec, "batch", True)
    try:
        _, G, dx = det_run(s, fill_nan, True)
        rep = tbl.Report("det-" + tbl._run_id((case, prec, "batch", True)))
        with torch.no_grad():
            tbl.check_forward(s, rep)
            tbl.check_backward(s, rep, [s.ws], [G], [dx])
        rep.print()
        assert not rep.fail, "\n".join(rep.fail[:40])
    finally:
        s.ws = None
        s.lib.wunet_destroy(s.ctx)


def test_workspace_query():
    """Without the flag the size is wunet_train_workspace_bytes_prec's; with it strictly larger; unknown bits give 0."""
    lib = _lib.load()
    for n, ci, shapes in ((12, 24, ((120, 16384), (3, 20480), (64, 16384))), (6, 20, ((5, 2048),)), (4, 8, ((2, 256),))):
        m = Model(n, ci)
        c = m._context(torch.device("cuda:0"))
        for B, T in shapes:
            for prec in (_lib.PREC_FP32, _lib.PREC_BF16):
                base = lib.wunet_train_workspace_bytes_prec(c, B, T, prec)
                assert base > 0
                for f in (0, _lib.TRAIN_FROZEN_BN, _lib.TRAIN_NO_PARAM_GRADS, _lib.TRAIN_FROZEN_BN | _lib.TRAIN_NO_PARAM_GRADS):
                    assert lib.wunet_train_workspace_bytes_ex(c, B, T, prec, f) == base
                    assert lib.wunet_train_workspace_bytes_ex(c, B, T, prec, f | DET) > base
                for bad in (4, 8, 32):
                    assert lib.wunet_train_workspace_bytes_ex(c, B, T, prec, bad) == 0
        m._release()


def test_workspace_sized_for_the_default_step_is_rejected():
    s = det_step("channel_plan", "fp32", "batch", True)
    try:
        with pytest.raises(_lib.WunetError, match="workspace too small"):
            _lib.check(s.forward_rc())                   # s.ws was sized without the flag
    finally:
        s.lib.wunet_destroy(s.ctx)


def test_naive_kernels_refuse_deterministic_mode(monkeypatch):
    """WUNET_TRAIN_NAIVE=1 (the one-thread-per-output cross-check) has no deterministic weight gradient: an error, never a
    silently non-repeatable step."""
    monkeypatch.setenv("WUNET_TRAIN_NAIVE", "1")
    s = det_step("channel_plan", "fp32", "batch", True)
    try:
        with pytest.raises(_lib.WunetError, match="deterministic"):
            det_run(s, fill_zeros, True)
    finally:
        s.ws = None
        s.lib.wunet_destroy(s.ctx)


SUBPROCESS_STEP = textwrap.dedent("""
    import hashlib, sys
    import numpy as np, torch
    sys.path.insert(0, sys.argv[1])
    from oracle import wunet_oracle as wo
    from wave_u_net_for_speech_enhancement_b200 import Model
    torch.backends.cudnn.deterministic = True
    n, ci, B, T = 12, 24, 4, 16384
    for prec in ("fp32", "bf16"):
        m = Model(n, ci, train_precision=prec)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in wo.make_state(n, ci, seed=31).items()})
        m = m.cuda().train()
        x = torch.from_numpy(wo.make_input(B, T, seed=32)).cuda().requires_grad_(True)
        y = m(x)
        (y * y).mean().backward()
        h = hashlib.sha256()
        for t in [y.detach(), x.grad] + [p.grad for p in m.parameters()] + [b for b in m.buffers()]:
            h.update(t.detach().contiguous().cpu().numpy().tobytes())
        print(prec, h.hexdigest())
""")


def test_step_is_repeatable_across_processes():
    digests = []
    for _ in range(2):
        r = subprocess.run([sys.executable, "-c", SUBPROCESS_STEP, ROOT], cwd=ROOT, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-3000:]
        digests.append(r.stdout.split())
    print(digests[0])
    assert len(digests[0]) == 4 and digests[0] == digests[1]


@pytest.mark.parametrize("golden", sorted(TRAIN_BARS))
def test_training_goldens(golden_dir, golden, monkeypatch):
    g = np.load(os.path.join(golden_dir, golden))
    n, ci, B, T = int(g["n_layers"]), int(g["channels_interval"]), int(g["B"]), int(g["T"])
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    noisy, clean = tbf.make_pair(B, T, int(g["pair_seed"]))
    ac = tbf.step_errors(tbf.make_model(n, ci, st, "torch"), g, noisy, clean, autocast=True)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    fp32 = tbf.step_errors(tbf.make_model(n, ci, st, "native", "fp32"), g, noisy, clean, autocast=False)
    bf16 = tbf.step_errors(tbf.make_model(n, ci, st, "native", "bf16"), g, noisy, clean, autocast=False)
    names = ("loss rel", "y max-abs", "worst grad rel", "running stats rel")
    for name, a, b, c, bar in zip(names, fp32, bf16, ac, TRAIN_BARS[golden]):
        av, bv, cv = (a[0], b[0], c[0]) if isinstance(a, tuple) else (a, b, c)
        print(f"{golden} {name}: deterministic fp32 {av:.2e}, deterministic bf16 {bv:.2e}, autocast {cv:.2e}, fp32 bar {bar:.0e}")
        assert av <= bar, (name, av, bar)
        assert bv <= max(2 * cv, bar), (name, bv, cv, bar)


@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("golden", [tag.SMALL, tag.FULL])
def test_autograd_goldens(golden_dir, golden, mode, monkeypatch):
    g, n, ci, st, noisy, clean = tag.load(golden_dir, golden)
    ac = tag.step_errors(tag.make_model(n, ci, st, mode, "torch"), g, st, mode, noisy, clean, autocast=True)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    fp32 = tag.step_errors(tag.make_model(n, ci, st, mode), g, st, mode, noisy, clean)
    bf16 = tag.step_errors(tag.make_model(n, ci, st, mode, "native", "bf16"), g, st, mode, noisy, clean)
    loss_bar, y_bar, grad_bar = AUTOGRAD_BARS[(golden, mode)]
    names = ("loss rel", "y max-abs", "worst grad rel", "dx rel", "running stats rel")
    for name, a, b, c, bar in zip(names, fp32, bf16, ac, (loss_bar, y_bar, grad_bar, grad_bar, 1e-5)):
        av, bv, cv = (a[0], b[0], c[0]) if isinstance(a, tuple) else (a, b, c)
        print(f"{golden} {mode} {name}: deterministic fp32 {av:.2e}, deterministic bf16 {bv:.2e}, autocast {cv:.2e}, bar {bar:.0e}")
        assert av <= bar, (name, av, bar)
        assert bv <= max(2 * cv, bar), (name, bv, cv, bar)


def adam_run(prec, B=4, T=16384, steps=30):
    torch.manual_seed(0)
    m = Model(12, 24, train_precision=prec).cuda().train()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    g = torch.Generator(device="cuda").manual_seed(1)
    clean = 0.1 * torch.randn(B, 1, T, device="cuda", generator=g)
    noisy = clean + 0.05 * torch.randn(B, 1, T, device="cuda", generator=g)
    losses = []
    for _ in range(steps):
        opt.zero_grad()
        loss = torch.nn.MSELoss()(clean, m(noisy))
        loss.backward()
        opt.step()
        losses.append(loss.detach())
    return torch.stack(losses).cpu(), {k: v.detach().clone() for k, v in m.state_dict().items()}


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("switch", ["cudnn", "algorithms"])
def test_thirty_adam_steps_repeat_bit_for_bit(prec, switch, monkeypatch):
    """What a user of the reference's trainer sees with "cudnn_deterministic": true: two 30-step Adam runs from the same
    state give the same losses and the same final state_dict, bit for bit."""
    if switch == "cudnn":
        monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    else:
        saved = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(True)
    try:
        (la, sa), (lb, sb) = adam_run(prec), adam_run(prec)
    finally:
        if switch != "cudnn":
            torch.use_deterministic_algorithms(saved)
    assert torch.isfinite(la).all()
    assert torch.equal(la, lb), (la - lb).abs().max()
    assert sa.keys() == sb.keys()
    diff = [k for k in sa if not torch.equal(sa[k], sb[k])]
    assert not diff, diff[:10]


@pytest.mark.parametrize("precision", ["bf16", "fp32_tc"])
def test_inference_forward_is_bitwise_repeatable(precision):
    n, ci, B, T = 12, 24, 256, 16384
    m = Model(n, ci, precision=precision)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in wo.make_state(n, ci, seed=41).items()})
    m = m.cuda().eval()
    x = torch.from_numpy(wo.make_input(B, T, seed=42)).cuda()
    with torch.no_grad():
        a = m(x).clone()
        b = m(x)
    assert torch.isfinite(a).all()
    assert torch.equal(a, b)
