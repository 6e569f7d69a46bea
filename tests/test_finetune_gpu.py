"""Fine-tuning with frozen layers in the native training step, on one H100: per-block BatchNorm modes and momenta, per-parameter
requires_grad (wunet_train_forward_blocks / wunet_train_backward_blocks).

1. Against the reference semantics: a float64 copy of the model through train_backend="torch" (it calls the BatchNorm modules
   themselves, so it honours their modes and momenta), at the state and batch of train_full_n12_c24_b2_t4096.npz. fp32 under
   test_train_gpu.py's bars (loss 1e-4 relative, y 1e-3, gradients 2e-2 of the largest entry, running statistics 1e-5);
   with every BatchNorm frozen the gradients under test_autograd_gpu.py's eval-mode bar (2e-5). bf16 / tf32 within max(2 x
   the error of PyTorch's own step at that precision in the same configuration, the fp32 bar), test_train_bf16_gpu.py's bar:
   the composite path under torch.autocast(bfloat16), or in fp32 with cuDNN's TF32 convolutions.
2. Deterministic mode, bit for bit at fp32, bf16 and tf32: .train() with every container in .eval() equals .eval() with
   eval_autograd="always"; partial requires_grad gives the full step's bits on every trainable gradient, y and the running
   buffers; the _blocks entry points with every block in training mode give the _ex bits; whole and split backward agree.
3. Early stop: with the encoder and the middle frozen and no dx, part 1 issues no kernel (torch.profiler); with dx the full
   chain runs and dx has the full step's bits.
4. A pass-through BatchNorm all-reduce hook with mixed modes is called only for batch-statistics blocks and changes no bit.
5. Two Adam steps through the data-parallel backward (split in two parts, masked gradient bucket) change no frozen parameter
   and no frozen running statistic."""
import ctypes
import os

import numpy as np
import pytest
import torch

import test_sync_bn_gpu as sbg
from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model, _lib
from wave_u_net_for_speech_enhancement_b200 import train_step as ts

pytestmark = [pytest.mark.gpu]

PRECS = ["fp32", "bf16", "tf32"]
FP32_BARS = (1e-4, 1e-3, 2e-2, 1e-5)         # loss relative, y max-abs, gradient relative to its largest entry, running stats
FROZEN_GRAD_REL = 2e-5
CASES = ["enc_mid_frozen", "alt_bn_frozen", "head_only", "momenta", "momentum_none"]


def golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "train_full_n12_c24_b2_t4096.npz"))
    n, ci, B, T = int(g["n_layers"]), int(g["channels_interval"]), int(g["B"]), int(g["T"])
    return n, ci, wo.make_state(n, ci, seed=int(g["state_seed"])), sbg.make_pair(B, T, int(g["pair_seed"]))


def make(n, ci, st, backend="native", prec="fp32", dtype=torch.float32, **kw):
    m = Model(n, ci, precision="fp32", train_backend=backend, train_precision=prec, **kw)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    return m.to(device="cuda:0", dtype=dtype).train()


def configure(m, case):
    bns = [blk[1] for blk in m._blocks()]
    if case == "enc_mid_frozen":
        for mod in (m.encoder, m.middle):
            mod.requires_grad_(False)
            for x in mod.modules():
                if isinstance(x, torch.nn.BatchNorm1d):
                    x.eval()
    elif case == "alt_bn_frozen":
        for i in range(0, len(bns), 2):
            bns[i].eval()
    elif case == "head_only":
        m.requires_grad_(False)
        m.out.requires_grad_(True)
        for bn in bns:
            bn.eval()
    elif case == "momenta":
        for i, bn in enumerate(bns):
            bn.momentum = 0.02 * (i + 1)
    elif case == "momentum_none":
        for bn in bns:
            bn.momentum = None
    return m


def run_steps(m, noisy, clean, steps=1):
    dt = next(m.parameters()).dtype
    x, c = torch.from_numpy(noisy).cuda().to(dt), torch.from_numpy(clean).cuda().to(dt)
    for _ in range(steps):
        m.zero_grad(set_to_none=True)
        y = m(x)
        loss = torch.nn.MSELoss()(c, y)
        loss.backward()
    return float(loss.detach()), y.detach().double()


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / max(float(b.double().abs().max()), 1e-30))


def errors(m, ref, loss, y, loss_ref, y_ref):
    """(loss relative, y max-abs, worst gradient relative, worst running statistic relative) of m against ref"""
    training = {k for k, mod in m.named_modules() if isinstance(mod, torch.nn.BatchNorm1d) and mod.training}
    g = 0.0
    for (k, p), (_, q) in zip(m.named_parameters(), ref.named_parameters()):
        assert (p.grad is None) == (q.grad is None) == (not p.requires_grad), k
        if p.grad is None:
            continue
        if k.endswith(".0.bias") and not k.startswith("out.") and k.replace(".0.bias", ".1") in training:
            continue                              # before batch-statistics BatchNorm: the gradient is rounding noise
        g = max(g, rel(p.grad, q.grad))
    s = max(rel(a, b) for (k, a), (_, b) in zip(m.state_dict().items(), ref.state_dict().items()) if "running" in k)
    for (k, a), (_, b) in zip(m.state_dict().items(), ref.state_dict().items()):
        if "num_batches" in k:
            assert int(a) == int(b), k
    return abs(loss - loss_ref) / loss_ref, float((y - y_ref).abs().max()), g, s


def torch_step_errors(n, ci, st, noisy, clean, case, prec, steps, ref_out, monkeypatch):
    """the error of PyTorch's own step at `prec` (the composite path) against float64, same configuration"""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", prec == "tf32")
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", prec == "tf32")
    m = configure(make(n, ci, st, "torch"), case)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=prec == "bf16"):
        out = run_steps(m, noisy, clean, steps)
    ref = ref_out[0]
    return errors(m, ref, *out, *ref_out[1:])


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("case", CASES)
def test_against_the_reference_semantics(golden_dir, monkeypatch, case, prec):
    if prec != "fp32" and case not in ("enc_mid_frozen", "head_only"):
        pytest.skip("bf16 / tf32: two masks")
    n, ci, st, (noisy, clean) = golden(golden_dir)
    steps = 2 if case == "momentum_none" else 1
    ref = configure(make(n, ci, st, "torch", dtype=torch.float64), case)
    m = configure(make(n, ci, st, prec=prec), case)
    ref_out = run_steps(ref, noisy, clean, steps)
    got = errors(m, ref, *run_steps(m, noisy, clean, steps), *ref_out)
    bars = list(FP32_BARS)
    if case == "head_only":
        bars[2] = FROZEN_GRAD_REL
    if case == "momentum_none":
        # the first step's factor is 1: the running statistics are the batch statistics themselves, not 0.1 of them over
        # exact pretrained values as under the 1e-5 bar (momentum 0.1), so that bar scales by 10
        bars[3] = 1e-4
    if prec != "fp32":
        base = torch_step_errors(n, ci, st, noisy, clean, case, prec, steps, (ref,) + ref_out, monkeypatch)
        bars = [max(2 * f, b) for f, b in zip(base, bars)]
    print(f"{case} {prec}: loss {got[0]:.2e} y {got[1]:.2e} grad {got[2]:.2e} running {got[3]:.2e} (bars {bars})")
    for name, v, b in zip(("loss", "y", "grad", "running"), got, bars):
        assert v <= b, (name, v, b)


def snapshot(m, y):
    out = {"y": y.clone()}
    out.update({"grad:" + k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None})
    out.update({k: v.clone() for k, v in m.state_dict().items() if "running" in k})
    return out


def bitwise(a, b, keys=None):
    keys = a.keys() if keys is None else keys
    diff = [k for k in keys if not torch.equal(a[k], b[k])]
    assert not diff, diff[:10]


@pytest.fixture
def deterministic(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)


@pytest.mark.parametrize("prec", PRECS)
def test_deterministic_bits(golden_dir, deterministic, monkeypatch, prec):
    n, ci, st, (noisy, clean) = golden(golden_dir)
    # .train() with every container in .eval() == .eval() with eval_autograd="always"
    a = make(n, ci, st, prec=prec)
    for blk in a._blocks():
        blk[1].eval()
    b = make(n, ci, st, prec=prec, eval_autograd="always").eval()
    sa, sb = (snapshot(m, run_steps(m, noisy, clean)[1]) for m in (a, b))
    bitwise(sa, sb)
    # partial requires_grad: the full step's bits on what it computes
    full = make(n, ci, st, prec=prec)
    sf = snapshot(full, run_steps(full, noisy, clean)[1])
    part = make(n, ci, st, prec=prec)
    part.encoder.requires_grad_(False)
    part.middle.requires_grad_(False)
    sp = snapshot(part, run_steps(part, noisy, clean)[1])
    assert len(sp) < len(sf)
    bitwise(sp, sf, sp.keys())
    # the _blocks entry points with every block in training mode == _ex
    blk = make(n, ci, st, prec=prec)
    nb = 2 * n + 1
    from wave_u_net_for_speech_enhancement_b200.unet_basic import _NativeTrainStep
    params = [t for q in blk._blocks() for t in (q[0].weight, q[0].bias, q[1].weight, q[1].bias)] + list(blk.out[0].parameters())
    x = torch.from_numpy(noisy).cuda()
    y = _NativeTrainStep.apply(blk, _lib.TRAIN_DETERMINISTIC, None, ([False] * nb, [0.1] * nb), x, *params)
    torch.nn.MSELoss()(torch.from_numpy(clean).cuda(), y).backward()
    for q in blk._blocks():
        q[1].num_batches_tracked += 1
    bitwise(snapshot(blk, y.detach().double()), sf)
    # whole == split (part 0, then part 1) backward, mixed modes and a partial mask, dx too
    outs = []
    for world in (1, 2):
        monkeypatch.setattr(ts, "data_parallel_world", lambda w=world: w)
        monkeypatch.setattr(ts.GradientBucket, "reduce_part", lambda self, k, group=None: None)
        m = configure(make(n, ci, st, prec=prec), "alt_bn_frozen")
        m.encoder.requires_grad_(False)
        xg = torch.from_numpy(noisy).cuda().requires_grad_(True)
        y = m(xg)
        torch.nn.MSELoss()(torch.from_numpy(clean).cuda(), y).backward()
        s = snapshot(m, y.detach())
        s["dx"] = xg.grad.clone()
        outs.append(s)
    bitwise(outs[0], outs[1])


class BlockRank(sbg.Rank):
    """test_sync_bn_gpu.Rank driving the _blocks entry points: per-block modes, momenta and a gradient mask (name -> bool
    per block for w, b, gamma, beta; wo, bo)"""

    def __init__(self, *a, frozen, momenta, mask, **kw):
        super().__init__(*a, **kw)
        self.frozen = (ctypes.c_ubyte * self.nb)(*frozen)
        self.momenta = (ctypes.c_float * self.nb)(*momenta)
        self.mask = mask

    def forward(self):
        P = self.ptrs
        return self.lib.wunet_train_forward_blocks(
            self.ctx, self.x.data_ptr(), self.y.data_ptr(), self.B, self.T, P(self.w), P(self.b), P(self.gamma), P(self.beta),
            P(self.rm), P(self.rv), self.wo.data_ptr(), self.bo.data_ptr(), 0.0, self.ws.data_ptr(), self.ws.numel() * 4,
            self.stream.cuda_stream, _lib.TRAIN_PRECISIONS[self.prec], self.flags, self.frozen, self.momenta)

    def backward(self, part=-1, dx=True):
        if part != 1:
            self.dy = (2.0 / (self.loss_frames * self.T)) * (self.y - self.clean)
        g = {k: (ctypes.c_void_p * self.nb)(*[t.data_ptr() if on else None for t, on in zip(self.G[k], self.mask[k])])
             for k in ("w", "b", "gamma", "beta")}
        head = [self.G[k].data_ptr() if self.mask[k] else None for k in ("wo", "bo")]
        return self.lib.wunet_train_backward_blocks(
            self.ctx, self.x.data_ptr(), self.y.data_ptr(), self.dy.data_ptr(), self.B, self.T, self.ptrs(self.w),
            self.ptrs(self.gamma), self.ptrs(self.beta), self.wo.data_ptr(), g["w"], g["b"], g["gamma"], g["beta"], head[0],
            head[1], self.ws.data_ptr(), self.ws.numel() * 4, self.stream.cuda_stream, self.dx.data_ptr() if dx else None, part,
            _lib.TRAIN_PRECISIONS[self.prec], self.flags, self.frozen)


def enc_mid_rank(n, ci, st, noisy, clean, prec, flags=_lib.TRAIN_DETERMINISTIC, frozen=None):
    nb = 2 * n + 1
    lower = [i <= n for i in range(nb)]
    mask = {k: [not f for f in lower] for k in ("w", "b", "gamma", "beta")}
    mask.update(wo=True, bo=True)
    return BlockRank(n, ci, st, noisy, clean, prec, flags, frozen=lower if frozen is None else frozen, momenta=[0.1] * nb,
                     mask=mask)


def cuda_kernels(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@pytest.mark.parametrize("prec", PRECS)
def test_early_stop(golden_dir, prec):
    n, ci, st, (noisy, clean) = golden(golden_dir)
    rk = enc_mid_rank(n, ci, st, noisy, clean, prec)
    nb = 2 * n + 1
    full = BlockRank(n, ci, st, noisy, clean, prec, _lib.TRAIN_DETERMINISTIC, frozen=[i <= n for i in range(nb)],
                     momenta=[0.1] * nb, mask={**{k: [True] * nb for k in ("w", "b", "gamma", "beta")}, "wo": True, "bo": True})
    try:
        with torch.cuda.stream(rk.stream):
            _lib.check(rk.forward())
            _lib.check(rk.backward(0, dx=False))
        rk.stream.synchronize()
        with torch.cuda.stream(rk.stream):
            k1 = cuda_kernels(lambda: _lib.check(rk.backward(1, dx=False)))
        assert k1 == [], k1[:10]
        # dx requested (and announced to part 0): the whole chain, with the full step's dx
        rk.step(parts=(0, 1))
        with torch.cuda.stream(rk.stream):
            k_dx = cuda_kernels(lambda: _lib.check(rk.backward(1, dx=True)))
        assert len(k_dx) > 2 * n
        full.step()
        rk.step()
        assert torch.equal(rk.dx, full.dx)
    finally:
        rk.close()
        full.close()


def test_sync_hook_only_for_batch_statistics_blocks(golden_dir):
    n, ci, st, (noisy, clean) = golden(golden_dir)
    nb = 2 * n + 1
    frozen = [i % 2 == 0 for i in range(nb)]
    a = enc_mid_rank(n, ci, st, noisy, clean, "fp32", frozen=frozen)
    b = enc_mid_rank(n, ci, st, noisy, clean, "fp32", frozen=frozen)
    counts = []
    try:
        _lib.check(a.install(lambda view: counts.append(view.numel())))
        a.step(parts=(0, 1))
        b.step(parts=(0, 1))
        batch = [i for i in range(nb) if not frozen[i]]
        widths = [a.lay[i]["Cout"] for i in batch]
        fwd = [c for w in widths for c in (w + 1, w)]
        bwd = [2 * a.lay[i]["Cout"] + 1 for i in sorted(batch, reverse=True)]
        assert counts == fwd + bwd
        assert torch.equal(a.y, b.y) and torch.equal(a.dx, b.dx)
        for i in range(nb):
            assert torch.equal(a.rm[i], b.rm[i]) and torch.equal(a.rv[i], b.rv[i])
            for k in ("w", "b", "gamma", "beta"):
                if a.mask[k][i]:
                    assert torch.equal(a.G[k][i], b.G[k][i]), (k, i)
                else:
                    assert torch.isnan(a.G[k][i]).all(), (k, i)              # a frozen slot is never written
    finally:
        a.install(None)
        a.close()
        b.close()


@pytest.mark.parametrize("prec", PRECS)
def test_two_adam_steps_leave_frozen_state_alone(golden_dir, monkeypatch, prec):
    n, ci, st, (noisy, clean) = golden(golden_dir)
    monkeypatch.setattr(ts, "data_parallel_world", lambda: 2)
    monkeypatch.setattr(ts.GradientBucket, "reduce_part", lambda self, k, group=None: None)
    m = configure(make(n, ci, st, prec=prec), "enc_mid_frozen")
    before = {k: v.clone() for k, v in m.state_dict().items()}
    opt = torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=1e-3)
    for _ in range(2):
        opt.zero_grad()
        run_steps(m, noisy, clean)
        opt.step()
    for k, v in m.state_dict().items():
        frozen = k.startswith(("encoder.", "middle."))
        assert torch.equal(v, before[k]) == frozen, k
