"""Synchronised BatchNorm statistics (nn.SyncBatchNorm) in the native training step, on one H100.

1. A pass-through hook (a world of one rank) reproduces the default step bit for bit: through Model and autograd with the
   ``_bn_allreduce`` seam, and through the C entry points with the split backward (part 0, then part 1).
2. Emulated ranks: R threads, each with its own context, stream and shard of the batch, drive the C entry points; the hook
   sums the ranks' buffers across the threads. (``loss.backward()`` cannot drive them: autograd runs every CUDA backward of
   a device on one worker thread, so two ranks blocking in each other's hook would deadlock.) They are compared with one
   context stepping the concatenated batch.
3. The float64 golden step at B = 2, split into two ranks of one frame: L = 1 per rank at the middle block, a shape only a
   synchronised step accepts.
4. A failing hook, and a buffer that is too small.
5. End to end: two processes (torchrun) over gloo on the same GPU, nn.SyncBatchNorm.convert_sync_batchnorm, loss.backward()
   and three Adam steps; an NCCL variant needs two GPUs."""
import ctypes
import os
import socket
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model, _lib

pytestmark = [pytest.mark.gpu]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRECS = ["fp32", "bf16", "tf32"]
MOMENTUM = 0.1
EPS = float(np.float32(1e-5))       # kBnEps as the kernels see it
REL = 1e-4                      # test_ddp_gpu.py's bar: y, gradients (relative to the largest entry)
# the float64 golden step's bars of the fp32 native step (test_train_deterministic_gpu.TRAIN_BARS): loss relative, y max-abs,
# worst gradient relative, running statistics relative
GOLDEN_BARS = (1e-4, 1e-3, 2e-2, 1e-5)


def make_pair(B, T, seed):
    g = np.random.Generator(np.random.PCG64(seed))
    clean = (0.1 * g.standard_normal((B, 1, T))).astype(np.float32)
    noisy = (clean + 0.05 * g.standard_normal((B, 1, T))).astype(np.float32)
    return noisy, clean


def ulp32(v):
    a = v.abs().float()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def within_ulp(got, want):
    """fp32 `got` within one fp32 ulp of the float64 `want`; -> (ok, number of values that differ from fp32(want))"""
    w = want.float()
    return bool(((got.double() - w.double()).abs() <= ulp32(w)).all()), int((got != w).sum())


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / max(float(b.double().abs().max()), 1e-30))


class Rank:
    """One data-parallel rank driving the C entry points: its own context, stream, parameters, running buffers, workspace,
    gradients and hook buffer."""

    def __init__(self, n, ci, st, noisy, clean, prec, flags=0, loss_frames=None):
        self.n, self.ci, self.prec, self.flags = n, ci, prec, flags
        self.B, _, self.T = noisy.shape
        self.loss_frames = loss_frames or self.B           # the loss is the mean over this many frames' samples
        self.nb = 2 * n + 1
        dev = torch.device("cuda:0")
        self.plan = wo.channel_plan(n, ci)
        t = lambda k: torch.from_numpy(np.asarray(st[k])).to(dev).contiguous()   # noqa: E731
        p = [q[0] for q in self.plan]
        self.w, self.b = [t(f"{k}.0.weight") for k in p], [t(f"{k}.0.bias") for k in p]
        self.gamma, self.beta = [t(f"{k}.1.weight") for k in p], [t(f"{k}.1.bias") for k in p]
        self.rm, self.rv = [t(f"{k}.1.running_mean") for k in p], [t(f"{k}.1.running_var") for k in p]
        self.wo, self.bo = t("out.0.weight"), t("out.0.bias")
        self.x, self.clean = torch.from_numpy(noisy).to(dev), torch.from_numpy(clean).to(dev)
        self.lib = _lib.load()
        self.ctx = ctypes.c_void_p()
        _lib.check(self.lib.wunet_create(n, ci, 0, ctypes.byref(self.ctx)))
        code = _lib.TRAIN_PRECISIONS[prec]
        nbytes = self.lib.wunet_train_workspace_bytes_ex(self.ctx, self.B, self.T, code, flags & ~_lib.TRAIN_NO_PARAM_GRADS)
        self.ws = torch.full((nbytes // 4,), float("nan"), dtype=torch.float32, device=dev)
        self.y = torch.full_like(self.x, float("nan"))
        self.dx = torch.full_like(self.x, float("nan"))
        self.bnbuf = torch.zeros(2 * n * ci + 1, dtype=torch.float64, device=dev)
        self.lay = [_lib.debug_train_layout(n, ci, self.B, self.T, i, prec) for i in range(self.nb)]
        self.stream = torch.cuda.Stream(dev)
        self.calls, self.errors, self.fn = 0, [], None
        nan = lambda ts: [torch.full_like(v, float("nan")) for v in ts]       # noqa: E731
        self.G = None if flags & _lib.TRAIN_NO_PARAM_GRADS else dict(
            w=nan(self.w), b=nan(self.b), gamma=nan(self.gamma), beta=nan(self.beta), wo=nan([self.wo])[0], bo=nan([self.bo])[0])

    def close(self):
        self.lib.wunet_destroy(self.ctx)

    def install(self, reducer, capacity=None):
        """reducer(view) sums the float64 view over the ranks in place (None: uninstall); -> the library's status"""
        if reducer is None:
            self.fn = None
            return self.lib.wunet_train_set_bn_allreduce(self.ctx, _lib.BN_ALLREDUCE_FN(), None, None, 0)

        def hook(user, ptr, count, stream):
            self.calls += 1
            try:
                assert stream == self.stream.cuda_stream
                off = (ptr - self.bnbuf.data_ptr()) // 8
                return int(reducer(self.bnbuf[off:off + count]) or 0)
            except BaseException as e:  # noqa: BLE001
                self.errors.append(e)
                return 1
        self.fn = _lib.BN_ALLREDUCE_FN(hook)
        cap = self.bnbuf.numel() if capacity is None else capacity
        return self.lib.wunet_train_set_bn_allreduce(self.ctx, self.fn, None, self.bnbuf.data_ptr(), cap)

    @staticmethod
    def ptrs(ts):
        return None if ts is None else (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])

    def forward(self):
        P = self.ptrs
        return self.lib.wunet_train_forward_ex(
            self.ctx, self.x.data_ptr(), self.y.data_ptr(), self.B, self.T, P(self.w), P(self.b), P(self.gamma), P(self.beta),
            P(self.rm), P(self.rv), self.wo.data_ptr(), self.bo.data_ptr(), MOMENTUM, self.ws.data_ptr(), self.ws.numel() * 4,
            self.stream.cuda_stream, _lib.TRAIN_PRECISIONS[self.prec], self.flags & ~_lib.TRAIN_NO_PARAM_GRADS)

    def backward(self, part=-1):
        P, g = self.ptrs, self.G or {}
        if part != 1:
            self.dy = (2.0 / (self.loss_frames * self.T)) * (self.y - self.clean)      # MSELoss(clean, y) of this rank
        return self.lib.wunet_train_backward_ex(
            self.ctx, self.x.data_ptr(), self.y.data_ptr(), self.dy.data_ptr(), self.B, self.T, P(self.w), P(self.gamma),
            P(self.beta), self.wo.data_ptr(), P(g.get("w")), P(g.get("b")), P(g.get("gamma")), P(g.get("beta")),
            g["wo"].data_ptr() if g else None, g["bo"].data_ptr() if g else None, self.ws.data_ptr(), self.ws.numel() * 4,
            self.stream.cuda_stream, self.dx.data_ptr() if part != 0 else None, part, _lib.TRAIN_PRECISIONS[self.prec],
            self.flags)

    def step(self, parts=(-1,), backward=True):
        """forward, then the backward in `parts`, on this rank's stream; raises on a failed call"""
        calls = [self.forward] + ([lambda p=p: self.backward(p) for p in parts] if backward else [])
        with torch.cuda.stream(self.stream):
            for call in calls:
                rc = call()
                if self.errors:
                    raise self.errors[0]
                _lib.check(rc)
        self.stream.synchronize()

    def view(self, i, field):
        d = self.lay[i]
        shape = (self.B, d["Cout"], d["L"]) if field in ("z", "act", "ga") else (d["Cout"],)
        o = d[field] // 4
        return self.ws[o:o + int(np.prod(shape))].view(shape)

    def grads(self):
        """name -> gradient, in the model's parameter names"""
        out = {}
        for i, q in enumerate(self.plan):
            for k, key in (("0.weight", "w"), ("0.bias", "b"), ("1.weight", "gamma"), ("1.bias", "beta")):
                out[f"{q[0]}.{k}"] = self.G[key][i]
        out["out.0.weight"], out["out.0.bias"] = self.G["wo"], self.G["bo"]
        return out


class Exchange:
    """Sums the ranks' buffers across threads (in rank order, so every rank gets the same doubles)."""

    def __init__(self, R):
        self.barrier = threading.Barrier(R, timeout=300)
        self.parts = [None] * R

    def reducer(self, r):
        def f(view):
            self.parts[r] = view.cpu()                     # after this rank's kernels (current stream = the rank's)
            self.barrier.wait()
            total = self.parts[0].clone()
            for p in self.parts[1:]:
                total += p
            self.barrier.wait()
            view.copy_(total)
        return f


def run_ranks(ranks, parts=(-1,), backward=True):
    ex = Exchange(len(ranks))
    for r, rk in enumerate(ranks):
        _lib.check(rk.install(ex.reducer(r)))
    errors = []

    def go(rk):
        try:
            rk.step(parts, backward)
        except BaseException as e:  # noqa: BLE001
            errors.append(e)
            ex.barrier.abort()
    th = [threading.Thread(target=go, args=(rk,)) for rk in ranks]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if errors:
        raise errors[0]


def make_ranks(n, ci, st, noisy, clean, shards, prec, flags):
    out, b = [], 0
    for s in shards:
        out.append(Rank(n, ci, st, noisy[b:b + s], clean[b:b + s], prec, flags))
        b += s
    return out


# ------------------------------------------------------------------------------------------------------------------------
# 1. pass-through hook == the default step, bit for bit
# ------------------------------------------------------------------------------------------------------------------------
def model_step(st, n, ci, prec, noisy, clean, seam, train=True):
    m = Model(n, ci, precision="fp32", train_precision=prec)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    m = m.cuda().train(train)
    if not train:
        for p in m.parameters():
            p.requires_grad_(True)
    calls = []
    if seam:
        m._bn_allreduce = lambda buf: calls.append(buf.numel())
    x = torch.from_numpy(noisy).cuda().requires_grad_(True)
    y = m(x)
    n_fwd = len(calls)
    torch.nn.MSELoss()(torch.from_numpy(clean).cuda(), y).backward()
    torch.cuda.synchronize()
    out = dict(y=y.detach(), dx=x.grad)
    out.update({k: p.grad for k, p in m.named_parameters()})
    out.update({k: v for k, v in m.state_dict().items() if "running" in k})
    return out, n_fwd, len(calls) - n_fwd


@pytest.mark.parametrize("prec", PRECS)
def test_passthrough_seam_reproduces_the_default_step(prec, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    n, ci, B, T = 12, 24, 3, 8192
    st = wo.make_state(n, ci, seed=11)
    noisy, clean = make_pair(B, T, 12)
    ref, _, _ = model_step(st, n, ci, prec, noisy, clean, seam=False)
    got, n_fwd, n_bwd = model_step(st, n, ci, prec, noisy, clean, seam=True)
    assert (n_fwd, n_bwd) == (2 * (2 * n + 1), 2 * n + 1)
    diff = [k for k in ref if not torch.equal(ref[k], got[k])]
    assert not diff, diff
    # eval-mode (frozen) BatchNorm never synchronises
    ref, _, _ = model_step(st, n, ci, prec, noisy, clean, seam=False, train=False)
    got, n_fwd, n_bwd = model_step(st, n, ci, prec, noisy, clean, seam=True, train=False)
    assert (n_fwd, n_bwd) == (0, 0)
    assert all(torch.equal(ref[k], got[k]) for k in ref)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("parts", [(-1,), (0, 1)], ids=["whole", "split"])
def test_passthrough_hook_reproduces_the_default_step_through_the_c_abi(prec, parts):
    n, ci, B, T = 12, 24, 3, 8192
    st = wo.make_state(n, ci, seed=13)
    noisy, clean = make_pair(B, T, 14)
    flags = _lib.TRAIN_DETERMINISTIC
    a, b = Rank(n, ci, st, noisy, clean, prec, flags), Rank(n, ci, st, noisy, clean, prec, flags)
    try:
        a.step(parts)
        _lib.check(b.install(lambda view: None))
        b.step(parts)
        assert b.calls == 2 * (2 * n + 1) + (2 * n + 1)
        for name in ("y", "dx", "rm", "rv", "G"):
            va, vb = getattr(a, name), getattr(b, name)
            if name == "G":
                va, vb = list(a.grads().values()), list(b.grads().values())
            for i, (u, v) in enumerate(zip(va if isinstance(va, list) else [va], vb if isinstance(vb, list) else [vb])):
                assert torch.equal(u, v), (name, i)
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------------------------------------------------------------
# 2. emulated ranks against one process on the concatenated batch
# ------------------------------------------------------------------------------------------------------------------------
RANK_CASES = ([(p, (2, 2), True) for p in PRECS] + [(p, (2, 2, 2), True) for p in PRECS] + [("fp32", (2, 2), False)] +
              [(p, (1, 3), True) for p in PRECS])


@pytest.mark.parametrize("prec, shards, pgrads", RANK_CASES,
                         ids=[f"{p}-{'+'.join(map(str, s))}" + ("" if g else "-no_param_grads") for p, s, g in RANK_CASES])
def test_emulated_ranks_match_the_concatenated_batch(prec, shards, pgrads):
    n, ci, T = 12, 24, 4096
    B = sum(shards)
    equal = len(set(shards)) == 1
    st = wo.make_state(n, ci, seed=17)
    noisy, clean = make_pair(B, T, 18)
    flags = 0 if pgrads else _lib.TRAIN_NO_PARAM_GRADS
    # equal shards: the single process takes the ranks' loss scale (mean over B / R frames), so both sides round the same dz
    # values to bf16 / tf32 operands; the sum of the ranks' gradients is then its gradient, R times the averaged one
    full = Rank(n, ci, st, noisy, clean, prec, flags, loss_frames=shards[0] if equal else None)
    ranks = make_ranks(n, ci, st, noisy, clean, shards, prec, flags)
    try:
        full.step(backward=equal)
        run_ranks(ranks, backward=equal)
        m = float(np.float32(MOMENTUM))                  # the kernels promote the fp32 momentum
        differing = {"mean": 0, "invstd": 0, "running": 0}
        for i in range(2 * n + 1):
            # the synchronised statistics against float64 from the ranks' own z: one fp32 ulp
            zs = [rk.view(i, "z").double() for rk in ranks]
            N = sum(z.shape[0] * z.shape[2] for z in zs)
            mu = sum(z.sum((0, 2)) for z in zs) / N
            var = sum(((z - mu[None, :, None]) ** 2).sum((0, 2)) for z in zs) / N
            rm = (1 - m) * full_rm0(st, full, i) + m * mu
            rv = (1 - m) * full_rv0(st, full, i) + m * var * (N / (N - 1))
            for rk in ranks:
                for name, got, want in (("mean", rk.view(i, "mean"), mu), ("invstd", rk.view(i, "invstd"), 1 / torch.sqrt(var + EPS)),
                                        ("running_mean", rk.rm[i], rm), ("running_var", rk.rv[i], rv)):
                    ok, _ = within_ulp(got, want)
                    assert ok, (i, name)
                assert torch.equal(rk.rm[i], ranks[0].rm[i]) and torch.equal(rk.rv[i], ranks[0].rv[i]), i
            # against the single process: one ulp where the blocks' z agree bit for bit, else 1e-4 of the channel's spread
            same_z = torch.equal(torch.cat([rk.view(i, "z") for rk in ranks]), full.view(i, "z"))
            for name, got, want in (("mean", ranks[0].view(i, "mean"), full.view(i, "mean")),
                                    ("invstd", ranks[0].view(i, "invstd"), full.view(i, "invstd")),
                                    ("running", ranks[0].rm[i], full.rm[i]), ("running", ranks[0].rv[i], full.rv[i])):
                differing[name] += int((got != want).sum())
                if same_z:
                    assert within_ulp(got, want.double())[0], (i, name)
                elif name == "mean":
                    assert float(((got - want).abs() * full.view(i, "invstd")).max()) <= REL, (i, name)
                else:
                    assert rel(got, want) <= REL, (i, name)
        y = torch.cat([rk.y for rk in ranks])
        print(f"{prec} shards {shards}: values differing from the single process {differing}, y rel {rel(y, full.y):.2e}")
        assert rel(y, full.y) <= REL
        if not equal:
            return                                       # per-rank mean losses weight unequal shards differently
        dx = torch.cat([rk.dx for rk in ranks])
        assert rel(dx, full.dx) <= REL, rel(dx, full.dx)
        if pgrads:
            worst = (0.0, "")
            gs = [rk.grads() for rk in ranks]
            for k, want in full.grads().items():
                if k.endswith(".0.bias") and not k.startswith("out."):
                    continue                             # conv bias ahead of BatchNorm: its gradient is rounding noise
                worst = max(worst, (rel(sum(g[k] for g in gs), want), k))
            print(f"{prec} shards {shards}: dx rel {rel(dx, full.dx):.2e}, worst summed gradient rel {worst[0]:.2e} ({worst[1]})")
            assert worst[0] <= REL, worst
    finally:
        for rk in [full] + ranks:
            rk.close()


def full_rm0(st, rk, i):
    return torch.from_numpy(np.asarray(st[f"{rk.plan[i][0]}.1.running_mean"])).cuda().double()


def full_rv0(st, rk, i):
    return torch.from_numpy(np.asarray(st[f"{rk.plan[i][0]}.1.running_var"])).cuda().double()


# ------------------------------------------------------------------------------------------------------------------------
# 3. the float64 golden step split over two ranks of one frame
# ------------------------------------------------------------------------------------------------------------------------
def test_golden_step_split_over_two_ranks(golden_dir):
    g = np.load(os.path.join(golden_dir, "train_full_n12_c24_b2_t4096.npz"))
    n, ci, B, T = int(g["n_layers"]), int(g["channels_interval"]), int(g["B"]), int(g["T"])
    assert B == 2 and T >> n == 1                        # one value per channel per rank at the middle block
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    noisy, clean = make_pair(B, T, int(g["pair_seed"]))
    ranks = make_ranks(n, ci, st, noisy, clean, (1, 1), "fp32", 0)
    try:
        run_ranks(ranks)
        y = torch.cat([rk.y for rk in ranks]).cpu().numpy()
        loss = float(np.mean((y.astype(np.float64) - clean) ** 2))
        worst = (0.0, "")
        gs = [rk.grads() for rk in ranks]
        for k in gs[0]:
            if k.endswith(".0.bias") and not k.startswith("out."):
                continue
            got = ((gs[0][k] + gs[1][k]) / 2).cpu().numpy().astype(np.float64)
            if "grad:" + k in g.files:
                e = float(np.abs(got - g["grad:" + k]).max() / max(np.abs(g["grad:" + k]).max(), 1e-30))
            else:
                norm = float(g["gnorm:" + k])
                e1 = abs(np.sqrt((got ** 2).sum()) - norm) / norm
                e2 = np.abs(got.reshape(-1)[g["gidx:" + k]] - g["gval:" + k]).max() / np.abs(got).max()
                e = float(max(e1, e2))
            worst = max(worst, (e, k))
        stat = 0.0
        for i, q in enumerate(ranks[0].plan):
            for buf, key in ((ranks[0].rm[i], "running_mean"), (ranks[0].rv[i], "running_var")):
                want = g[f"stat:{q[0]}.1.{key}"]
                stat = max(stat, float(np.abs(buf.cpu().numpy() - want).max() / max(np.abs(want).max(), 1e-30)))
        errs = (abs(loss - float(g["loss"])) / float(g["loss"]), float(np.abs(y - g["y"]).max()), worst[0], stat)
        print("golden split over two ranks of B = 1: loss rel %.2e, y max-abs %.2e, worst grad rel %.2e (%s), running rel %.2e"
              % (errs[0], errs[1], worst[0], worst[1], errs[3]))
        for e, bar in zip(errs, GOLDEN_BARS):
            assert e <= bar, (errs, GOLDEN_BARS)
    finally:
        for rk in ranks:
            rk.close()


# ------------------------------------------------------------------------------------------------------------------------
# 4. failures
# ------------------------------------------------------------------------------------------------------------------------
def test_failing_hook_and_small_buffer():
    n, ci, B, T = 4, 8, 2, 256
    st = wo.make_state(n, ci, seed=3)
    noisy, clean = make_pair(B, T, 4)
    rk = Rank(n, ci, st, noisy, clean, "fp32", 0)
    try:
        assert rk.install(lambda v: None, capacity=2 * n * ci) == -1                 # WUNET_EINVAL
        assert "too small" in rk.lib.wunet_last_error().decode()
        assert rk.lib.wunet_train_set_bn_allreduce(rk.ctx, _lib.BN_ALLREDUCE_FN(lambda *a: 0), None, None, 65) == -1
        # the forward fails at block 1's sums: nothing after the hook is enqueued
        _lib.check(rk.install(lambda v: 7 if rk.calls == 3 else 0))
        with torch.cuda.stream(rk.stream):
            assert rk.forward() == -2                                                 # WUNET_ECUDA
        msg = rk.lib.wunet_last_error().decode()
        assert "block 1" in msg and "status 7" in msg, msg
        rk.stream.synchronize()
        assert rk.calls == 3 and not torch.isnan(rk.view(0, "mean")).any()
        assert torch.isnan(rk.view(1, "mean")).all() and torch.isnan(rk.view(2, "z")).all() and torch.isnan(rk.y).all()
        # the backward fails at its first block (the last decoder): no weight gradient, no dx
        _lib.check(rk.install(lambda v: None))
        rk.step(backward=False)
        _lib.check(rk.install(lambda v: 1))
        with torch.cuda.stream(rk.stream):
            assert rk.backward() == -2
        assert f"block {2 * n}" in rk.lib.wunet_last_error().decode()
        rk.stream.synchronize()
        assert torch.isnan(rk.G["w"][2 * n]).all() and torch.isnan(rk.dx).all()
        assert rk.install(None) == 0
        rk.step()                                       # uninstalled: the default step again
        assert torch.isfinite(rk.dx).all()
    finally:
        rk.close()


def test_model_reraises_the_reducer_exception():
    m = Model(4, 8, precision="fp32").cuda().train()

    def bad(buf):
        raise KeyError("reducer")
    m._bn_allreduce = bad
    with pytest.raises(KeyError):
        m(torch.zeros(2, 1, 256, device="cuda"))
    m._bn_allreduce = None
    m(torch.zeros(2, 1, 256, device="cuda")).sum().backward()          # the hook was removed
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------------
# 5. end to end: torchrun, nn.SyncBatchNorm.convert_sync_batchnorm, loss.backward(), Adam
# ------------------------------------------------------------------------------------------------------------------------
WORKER = r'''
import os, sys
sys.path.insert(0, os.environ["WUNET_ROOT"])
import numpy as np, torch, torch.distributed as dist, torch.nn as nn
from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model
from wave_u_net_for_speech_enhancement_b200.train_step import train_step
backend = os.environ["SYNC_BN_BACKEND"]
rank = int(os.environ["LOCAL_RANK"])
dev = torch.device("cuda", rank if backend == "nccl" else 0)          # gloo: both ranks on one GPU
torch.cuda.set_device(dev)
dist.init_process_group(backend, device_id=dev if backend == "nccl" else None)
world = dist.get_world_size()
n, ci, Bl, T, lr = 12, 24, 2, 4096, 1e-3
st = {k: torch.from_numpy(np.asarray(v)) for k, v in wo.make_state(n, ci, seed=2).items()}
g = np.random.Generator(np.random.PCG64(50))
clean = (0.1 * g.standard_normal((world * Bl, 1, T))).astype(np.float32)
noisy = (clean + 0.05 * g.standard_normal((world * Bl, 1, T))).astype(np.float32)
clean, noisy = torch.from_numpy(clean).to(dev), torch.from_numpy(noisy).to(dev)
sl = slice(rank * Bl, (rank + 1) * Bl)
mse = torch.nn.MSELoss()
def make(sync):
    m = Model(n, ci, precision="fp32", data_parallel="auto" if sync else "off")
    m.load_state_dict(st)
    if sync:
        m = nn.SyncBatchNorm.convert_sync_batchnorm(m)
    return m.to(dev).train()
def rel(a, b):
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)
def running(m):
    return {k: v for k, v in m.state_dict().items() if "running" in k}
def same_on_every_rank(ts):
    flat = torch.cat([t.detach().reshape(-1).float() for t in ts])
    flat = flat if backend == "nccl" else flat.cpu()
    got = [torch.zeros_like(flat) for _ in range(world)]
    dist.all_gather(got, flat)
    return all(torch.equal(got[0], t) for t in got)
# one step: this rank's shard with synchronised statistics, against one process on the concatenated batch
ms, mr = make(True), make(False)
assert ms.reduces_gradients
ys = ms(noisy[sl]); mse(clean[sl], ys).backward()
yr = mr(noisy); mse(clean, yr).backward()
assert rel(ys.detach(), yr.detach()[sl]) <= 1e-4
worst = max((rel(a.grad, b.grad), k) for (k, a), b in zip(ms.named_parameters(), mr.parameters())
            if not (k.endswith(".0.bias") and not k.startswith("out.")))
assert worst[0] <= 1e-4, worst
rs, rr = running(ms), running(mr)
wrun = max(rel(rs[k], rr[k]) for k in rr)
assert wrun <= 1e-5, wrun
assert same_on_every_rank(list(rs.values())), "running statistics differ across ranks"
# three Adam steps through the public step
ms, mr = make(True), make(False)
os_, or_ = (torch.optim.Adam(m.parameters(), lr=lr, betas=(0.9, 0.999)) for m in (ms, mr))
for _ in range(3):
    train_step(ms, os_, mse, noisy[sl], clean[sl])
    or_.zero_grad(); mse(clean, mr(noisy)).backward(); or_.step()
assert same_on_every_rank(list(ms.parameters()) + list(running(ms).values())), "replicas diverged"
# Adam turns rounding-noise gradient entries into +-lr steps (test_train_gpu.py): 3 steps x 2 lr apart at most
dparam = max(float((a - b).abs().max()) for a, b in zip(ms.parameters(), mr.parameters()))
assert dparam <= 3 * 2 * lr * 1.05, dparam
wrun3 = max(rel(running(ms)[k], v) for k, v in running(mr).items())
assert wrun3 <= 1e-3, wrun3
if rank == 0:
    print("SYNC_BN_OK %s: worst gradient rel %.2e (%s), running rel %.2e; after 3 Adam steps: parameters %.2e apart, "
          "running rel %.2e" % (backend, worst[0], worst[1], wrun, dparam, wrun3))
dist.destroy_process_group()
'''


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_two_process_sync_batchnorm(tmp_path, backend):
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    env = dict(os.environ, WUNET_ROOT=ROOT, SYNC_BN_BACKEND=backend)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)],
                         env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    assert "SYNC_BN_OK" in out.stdout
    print(out.stdout.strip().splitlines()[-1])
