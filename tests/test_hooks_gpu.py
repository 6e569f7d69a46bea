"""Forward hooks on the block containers (encoder[i], encoder[i].main, middle, decoder[j], decoder[j].main, out) with the
native forward, on an H100.

Eval forward (wunet_forward_export): the hooked outputs match the reference's own hooks (tests/golden/*.npz, recorded by
oracle/gen_golden.py with forward hooks on the live reference module) at the per-level bars of test_parity_gpu.py, equal
read_level bit for bit, and leave y and the launch count unchanged. Training (wunet_train_backward_inject): a feature loss on
hooked levels gives the gradients of the composite path (train_backend="torch") in float64, at the bars of
test_autograd_gpu.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model, _lib

pytestmark = pytest.mark.gpu

FP32_TOL = 1e-4            # test_parity_gpu.py: fp32 and fp32_tc, max-abs
HALF_LEVEL_REL = 8e-3      # test_parity_gpu.py BF16_LEVEL_REL: max-abs error over max-abs level (bf16; fp16 is tighter)


def make_model(n, ci, st, precision="fp32_tc", **kw):
    m = Model(n, ci, precision=precision, **kw)
    m.load_state_dict({k: v if torch.is_tensor(v) else torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    return m.to("cuda:0")


def containers(m):
    n = m.n_layers
    cs = []
    for i in range(n):
        cs += [(f"encoder.{i}.main", m.encoder[i].main, i), (f"encoder.{i}", m.encoder[i], i)]
    cs.append(("middle", m.middle, n))
    for j in range(n):
        cs += [(f"decoder.{j}.main", m.decoder[j].main, n + 1 + j), (f"decoder.{j}", m.decoder[j], n + 1 + j)]
    cs.append(("out", m.out, 2 * n + 1))
    return cs


def hook_all(m, which=None):
    """Register a recording hook on every container (or the names in `which`): -> (record list, handles)."""
    rec, hs = [], []
    for name, mod, b in containers(m):
        if which is None or name in which:
            hs.append(mod.register_forward_hook(lambda mod, args, out, name=name, b=b: rec.append((name, b, args, out))))
    return rec, hs


def levels_of(rec):
    return {b: out for name, b, args, out in rec if not name.endswith(".main") and name != "out"}


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc", "fp16", "bf16"])
def test_hooks_match_the_reference_hooks(golden_dir, precision):
    """Every container fires once, in the reference's order, with the reference's input and output; the outputs match the
    reference's own hook records: every level of small_n4_c8 in full, the probes of full_n12_c24_b2 (and abssum at fp32)."""
    g = np.load(f"{golden_dir}/small_n4_c8.npz")
    n, ci, T, B = int(g["n_layers"]), int(g["channels_interval"]), int(g["T"]), int(g["B"])
    m = make_model(n, ci, wo.make_state(n, ci, seed=int(g["state_seed"])), precision).eval()
    x = torch.from_numpy(wo.make_input(B, T, seed=int(g["input_seed"]))).cuda()
    rec, hs = hook_all(m)
    with torch.no_grad():
        y = m(x)
    assert [r[0] for r in rec] == [c[0] for c in containers(m)]
    lv = levels_of(rec)
    for name, b, args, out in rec:
        if name == "out":
            assert out is y
            assert torch.equal(args[0], torch.cat([lv[2 * n], x], 1))
            continue
        ref = g[f"level_{b}"]
        got = out.cpu().numpy()
        err = np.abs(got - ref).max()
        bar = FP32_TOL if precision in ("fp32", "fp32_tc") else HALF_LEVEL_REL * np.abs(ref).max()
        assert err <= bar, (name, err, bar)
        want_in = x if b == 0 else lv[b - 1][:, :, ::2] if b <= n else torch.cat(
            [F.interpolate(lv[b - 1], scale_factor=2, mode="linear", align_corners=True), lv[2 * n - b]], 1)
        assert torch.equal(args[0], want_in), name
    for h in hs:
        h.remove()

    full = np.load(f"{golden_dir}/full_n12_c24_b2.npz")
    m = make_model(12, 24, wo.make_state(12, 24, seed=0), precision).eval()
    x = torch.from_numpy(wo.make_input(2, 16384, seed=int(full["input_seed"]))).cuda()
    rec, _ = hook_all(m)
    with torch.no_grad():
        m(x)
    for b, out in levels_of(rec).items():
        got = out.cpu().numpy()
        probe = full[f"probe_{b}"]
        err = np.abs(got[0][:, full[f"probe_idx_{b}"]] - probe).max()
        bar = FP32_TOL if precision in ("fp32", "fp32_tc") else HALF_LEVEL_REL * np.abs(probe).max()
        assert err <= bar, (b, err, bar)
        if precision == "fp32":
            a = np.abs(got.astype(np.float64)).sum()
            assert abs(a - float(full[f"abssum_{b}"])) <= 1e-5 * a + 1e-2, b


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc", "fp16", "bf16"])
@pytest.mark.parametrize("n,ci,B,T", [(12, 24, 2, 16384), (12, 48, 1, 16384), (10, 64, 257, 4096), (4, 8, 3, 256)])
def test_hooked_levels_are_read_level_bit_for_bit(monkeypatch, precision, n, ci, B, T):
    """Levels equal read_level (decoder[n-1]: read_level of a context that stores it, WUNET_TC_STORE_LAST=1); y and the launch
    count are those of the forward without hooks, and removing the hooks restores exactly that forward."""
    st = wo.make_state(n, ci, seed=7)
    x = torch.from_numpy(wo.make_input(B, T, seed=8)).cuda()
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "0")
    m = make_model(n, ci, st, precision).eval()
    with torch.no_grad():
        y0 = m(x)
        launches = m.last_launch_count()
        rec, hs = hook_all(m)
        y1 = m(x)
        assert m.last_launch_count() == launches
        lv = levels_of(rec)
        assert torch.equal(y0, y1)
        for b in range(2 * n):
            assert torch.equal(lv[b], m.read_level(b, B, T)), b
        for h in hs:
            h.remove()
        y2 = m(x)
        assert m.last_launch_count() == launches and torch.equal(y2, y0)
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")
    m2 = make_model(n, ci, st, precision).eval()
    with torch.no_grad():
        assert torch.equal(m2(x), y0)
        assert torch.equal(lv[2 * n], m2.read_level(2 * n, B, T))


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc", "bf16"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_model_levels_are_the_float_levels_rounded_once(precision, dtype):
    n, ci, B, T = 12, 24, 2, 16384
    st = wo.make_state(n, ci, seed=3)
    x16 = torch.from_numpy(wo.make_input(B, T, seed=4)).cuda().to(dtype)
    m16 = make_model(n, ci, st, precision).eval().to(dtype)
    m32 = make_model(n, ci, {k: v.to(torch.float32) if v.is_floating_point() else v for k, v in m16.state_dict().items()},
                     precision).eval()                       # the half model's parameters, widened
    r32, _ = hook_all(m32, {"encoder.0", "middle", f"decoder.{n - 1}", "out"})
    r16, _ = hook_all(m16, {"encoder.0", "middle", f"decoder.{n - 1}", "out"})
    with torch.no_grad():
        y32, y16 = m32(x16.float()), m16(x16)
    assert torch.equal(y16, y32.to(dtype))
    for a, b in zip(r32, r16):
        assert b[3].dtype == dtype and torch.equal(b[3], a[3].to(dtype)), a[0]


# ------------------------------------------------------------------------------------------------------------------------------
# training: gradients through the hooked levels
# ------------------------------------------------------------------------------------------------------------------------------
def feature_step(m, noisy, clean, targets, weights, dtype=torch.float32, x_grad=True):
    """loss = mse(y, clean) + sum_k w_k mse(level_k, target_k) through hooks; -> (loss, y, dx, the levels)."""
    feats = {}
    hs = [m.decoder[b - m.n_layers - 1] if b > m.n_layers else (m.middle if b == m.n_layers else m.encoder[b]) for b in targets]
    handles = [h.register_forward_hook(lambda mod, a, out, b=b: feats.__setitem__(b, out)) for h, b in zip(hs, targets)]
    x = torch.from_numpy(noisy).cuda().to(dtype).requires_grad_(x_grad)
    y = m(x)
    loss = F.mse_loss(y, torch.from_numpy(clean).cuda().to(dtype))
    for b, t in targets.items():
        loss = loss + weights[b] * F.mse_loss(feats[b], t.to(dtype))
    loss.backward()
    for h in handles:
        h.remove()
    return float(loss.detach()), y.detach(), None if x.grad is None else x.grad.detach().double(), feats


def worst_grad(a, b, skip_noise):
    worst = (0.0, "")
    for (k, p), q in zip(a.named_parameters(), b.parameters()):
        if p.grad is None or (skip_noise and k.endswith(".0.bias") and not k.startswith("out.")):
            continue
        d = (p.grad.double() - q.grad.double()).abs().max() / q.grad.double().abs().max().clamp_min(1e-30)
        worst = max(worst, (float(d), k))
    return worst


def setup_small(seed=21):
    n, ci, B, T = 4, 8, 3, 256
    st = wo.make_state(n, ci, seed=seed)
    g = np.random.Generator(np.random.PCG64(seed + 1))
    clean = (0.1 * g.standard_normal((B, 1, T))).astype(np.float32)
    noisy = (clean + 0.05 * g.standard_normal((B, 1, T))).astype(np.float32)
    # a mix of encoder, middle and decoder levels, with targets near the levels' scale
    shapes = {1: (B, 2 * ci, T // 2), n: (B, n * ci, T >> n), n + 2: (B, (n - 1) * ci, T >> (n - 2)), 2 * n: (B, ci, T)}
    targets = {b: torch.from_numpy(0.5 * g.standard_normal(s).astype(np.float32)).cuda() for b, s in shapes.items()}
    weights = {1: 0.3, n: 0.2, n + 2: 0.5, 2 * n: 1.0}
    return n, ci, st, noisy, clean, targets, weights


@pytest.mark.parametrize("train_precision", ["fp32", "bf16", "fp16_scaled"])
@pytest.mark.parametrize("mode", ["train", "eval"])
def test_feature_loss_gradients_match_the_composite_path(train_precision, mode, monkeypatch):
    """Native step with a feature loss on four levels against the composite path in float64 (truth) and, for the 16-bit
    training precisions, under bf16 autocast in fp32 (their bar: twice autocast's error, at least the fp32 bar, as in
    test_train_bf16_gpu.py). Eval mode is fine-tuning with eval_autograd="always" (frozen BatchNorm statistics)."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    n, ci, st, noisy, clean, targets, weights = setup_small()
    kw = {"eval_autograd": "always"} if mode == "eval" else {}
    nat = make_model(n, ci, st, "fp32", train_backend="native", train_precision=train_precision, **kw).train(mode == "train")
    ref = make_model(n, ci, st, "fp32", train_backend="torch", **kw).train(mode == "train").double()
    l_n, y_n, dx_n, f_n = feature_step(nat, noisy, clean, targets, weights)
    l_r, y_r, dx_r, f_r = feature_step(ref, noisy, clean, targets, weights, torch.float64)
    bar = 2e-4                                                  # test_autograd_gpu.py FP32_BARS, small config
    if train_precision != "fp32":
        ac = make_model(n, ci, st, "fp32", train_backend="torch", **kw).train(mode == "train")
        with torch.autocast("cuda", torch.bfloat16):
            feature_step(ac, noisy, clean, targets, weights)
        bar = max(bar, 2 * worst_grad(ac, ref, mode == "train")[0])
    for b in targets:
        assert f_n[b].dtype == torch.float32 and f_n[b].requires_grad
    worst = worst_grad(nat, ref, mode == "train")
    dx = float((dx_n - dx_r).abs().max() / dx_r.abs().max())
    print(f"{train_precision} {mode}: loss rel {abs(l_n - l_r) / l_r:.2e}, worst grad {worst[0]:.2e} ({worst[1]}), dx {dx:.2e}, "
          f"bar {bar:.1e}")
    assert worst[0] <= bar, worst
    assert dx <= bar, dx


def test_feature_loss_changes_the_gradients():
    """The injected gradient is not lost: without the feature terms the gradients differ."""
    n, ci, st, noisy, clean, targets, weights = setup_small()
    a = make_model(n, ci, st, "fp32").train()
    b = make_model(n, ci, st, "fp32").train()
    feature_step(a, noisy, clean, targets, weights)
    feature_step(b, noisy, clean, targets, {k: 0.0 * v for k, v in weights.items()})
    assert worst_grad(a, b, True)[0] > 1e-2


def test_deterministic_step_is_bitwise_repeatable_with_injections(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    n, ci, st, noisy, clean, targets, weights = setup_small()
    runs = []
    for _ in range(2):
        m = make_model(n, ci, st, "fp32", train_precision="bf16").train()
        _, y, dx, _ = feature_step(m, noisy, clean, targets, weights)
        runs.append((y, dx, [p.grad.clone() for p in m.parameters()]))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    assert all(torch.equal(a, b) for a, b in zip(runs[0][2], runs[1][2]))


def test_frozen_encoder_with_a_decoder_feature_loss(monkeypatch):
    """model.encoder.requires_grad_(False) and a loss on decoder levels only: the encoders get no gradient, the rest matches
    the composite path in float64; the early stop of the per-block backward still holds."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    n, ci, st, noisy, clean, targets, weights = setup_small()
    dec = {b: t for b, t in targets.items() if b > n}
    nat = make_model(n, ci, st, "fp32").train()
    ref = make_model(n, ci, st, "fp32", train_backend="torch").train().double()
    for m in (nat, ref):
        m.encoder.requires_grad_(False)
    feature_step(nat, noisy, clean, dec, weights, x_grad=False)
    feature_step(ref, noisy, clean, dec, weights, torch.float64, x_grad=False)
    assert all(p.grad is None for p in nat.encoder.parameters())
    worst = worst_grad(nat, ref, True)
    assert worst[0] <= 2e-4, worst


def test_split_backward_places_each_injection_in_its_part():
    """The two-part backward of data-parallel training (part 0: head + decoders, part 1: middle + encoders) with injections
    into an encoder, the middle and decoders equals the whole backward bit for bit (C ABI, batch statistics, deterministic
    mode: without it the weight gradients' float atomics differ from run to run)."""
    import ctypes
    n, ci, st, noisy, clean, targets, weights = setup_small()
    m = make_model(n, ci, st, "fp32").train()
    lib = _lib.load()
    B, T = noisy.shape[0], noisy.shape[2]
    x = torch.from_numpy(noisy).cuda()
    blocks = m._blocks()
    keep = []

    def ptr(ts):
        keep.append(ts)
        return (ctypes.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])

    c = m._context(x.device)
    det = _lib.TRAIN_DETERMINISTIC
    ws = torch.empty(lib.wunet_train_workspace_bytes_ex(c, B, T, 0, det), dtype=torch.uint8, device="cuda")
    y = torch.empty_like(x)
    rm, rv = [b[1].running_mean.clone() for b in blocks], [b[1].running_var.clone() for b in blocks]
    cw, cb = [b[0].weight for b in blocks], [b[0].bias for b in blocks]
    bw, bb = [b[1].weight for b in blocks], [b[1].bias for b in blocks]
    _lib.check(lib.wunet_train_forward_ex(c, x.data_ptr(), y.data_ptr(), B, T, ptr(cw), ptr(cb), ptr(bw), ptr(bb), ptr(rm),
                                          ptr(rv), m.out[0].weight.data_ptr(), m.out[0].bias.data_ptr(), 0.1, ws.data_ptr(),
                                          ws.numel(), None, 0, det))
    gy = torch.randn_like(y)
    g_act = [None] * (2 * n + 1)
    for b, t in targets.items():
        g_act[b] = torch.randn_like(t)

    def backward(parts):
        grads = [[torch.empty_like(t) for t in ts] for ts in (cw, cb, bw, bb)]
        go = [torch.empty_like(m.out[0].weight), torch.empty_like(m.out[0].bias)]
        dx = torch.empty_like(x)
        wsc = ws.clone()
        for part in parts:
            _lib.check(lib.wunet_train_backward_inject(
                c, x.data_ptr(), y.data_ptr(), gy.data_ptr(), B, T, ptr(cw), ptr(bw), ptr(bb), m.out[0].weight.data_ptr(),
                *[ptr(g) for g in grads], go[0].data_ptr(), go[1].data_ptr(), wsc.data_ptr(), wsc.numel(), None,
                dx.data_ptr(), part, 0, det, None, ptr(g_act)))
        torch.cuda.synchronize()
        return [t for g in grads for t in g] + go + [dx]

    whole, split = backward((-1,)), backward((0, 1))
    assert all(torch.equal(a, b) for a, b in zip(whole, split))
    g_act[:] = [None] * len(g_act)
    plain = backward((-1,))
    assert not torch.equal(plain[-1], whole[-1])                # the injections reached dx


# ------------------------------------------------------------------------------------------------------------------------------
# refusals and global hooks on the device path
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("train", [False, True])
def test_refusals_raise_on_the_device_path(train):
    n, ci = 4, 8
    m = make_model(n, ci, wo.make_state(n, ci, seed=1), "fp32").train(train)
    x = torch.from_numpy(wo.make_input(2, 256, seed=2)).cuda()
    cases = [
        (lambda: m.decoder[1].register_forward_pre_hook(lambda *a: None), NotImplementedError, "decoder.1"),
        (lambda: m.encoder[2].main[0].register_forward_hook(lambda *a: None), NotImplementedError, "encoder.2.main.0"),
        (lambda: m.middle.register_full_backward_hook(lambda *a: None), NotImplementedError, "middle"),
        (lambda: m.out[1].register_full_backward_pre_hook(lambda *a: None), NotImplementedError, "out.1"),
        (lambda: m.encoder[0].register_forward_hook(lambda mod, a, o: o * 2), RuntimeError, "encoder.0"),
    ]
    for reg, exc, name in cases:
        h = reg()
        with pytest.raises(exc, match=name.replace(".", r"\.")):
            m(x)
        h.remove()
    m(x)


def test_global_forward_hooks_fire_on_the_containers():
    n, ci = 4, 8
    m = make_model(n, ci, wo.make_state(n, ci, seed=1), "bf16").eval()
    x = torch.from_numpy(wo.make_input(2, 256, seed=2)).cuda()
    seen = []
    h = torch.nn.modules.module.register_module_forward_hook(lambda mod, a, o: seen.append(mod))
    try:
        with torch.no_grad():
            m(x)
    finally:
        h.remove()
    assert seen[:-1] == [c[1] for c in containers(m)] and seen[-1] is m
