"""Teacher-forced check of every kernel of the native training step (csrc/wunet_train.cu; csrc/wunet_train_tc.cu at bf16 and
tf32, csrc/wunet_train_tc_f16.cu at fp16_scaled), block by block, against float64.

The step runs through wunet_train_forward_ex / wunet_train_backward_ex (the "blocks" runs: wunet_train_forward_blocks /
wunet_train_backward_blocks, with per-block BatchNorm modes and momenta and null gradient slots) on a workspace this test
allocates; every block's
tensors are read as views given by the host-only layout query (wunet_debug_train_layout). For each block, what its kernels
should have produced is recomputed in float64 on the GPU **from the native inputs of that block**: the block input is built
from the native activations, the BatchNorm backward starts from an activation gradient routed (in float64) from the native
dz of the blocks that consume this one. Errors therefore do not compound over 25 blocks, and each kernel is held to a bar
that fits its own arithmetic:

- convolution-shaped outputs (z, the input gradients routed into da, dx): |err| <= CONV_REL * sum |products| of that output.
  A wrong tap, channel or frame offset moves an output by about sum |products| / sqrt(products) >= 1e-2 of that sum.
- weight gradients: |err| <= WGRAD_REL * sum |products|, a sum over B * L positions; see WGRAD_REL.
- elementwise outputs replayed in the kernels' own fp32 order (BatchNorm + LeakyReLU) and double reductions rounded once to
  fp32 (BatchNorm statistics, running buffers, conv bias gradient): 1 fp32 ulp, plus 1e-12 of the sum of magnitudes for the
  sums whose value can be cancellation noise.
- dz: the bar of the routed activation gradient propagated through the BatchNorm backward, plus its own fp32 roundings.
- the head (1x1 conv + tanh) and its gradients (warp sums + atomicAdd over B * T samples): see HEAD_REL.
In bf16, tf32 and fp16_scaled mode the reference convolves the operands the kernels multiply, rounded as they round them
(bf16: nearest even; tf32: cvt.rna, nearest with ties away from zero; fp16: nearest even, subnormals kept), block by block as
the layout query reports the block's kernels. An interpolated operand (decoder input) is computed in fp32 first; the kernel's
value may differ from the exactly rounded one by its own rounding (|err| <= 2^-23 of |lam0 a| + |lam1 b|), and where that
interval straddles a rounding boundary the operand may round to the other neighbour: the bar adds that interval, weighted like
the products it enters.

fp16_scaled: the forward operands are not scaled; the input- and weight-gradient passes multiply f16(dz 2^k) 2^-k, with k of
the block's max |dz|. The block's scale slot (field 22 of the layout query) must hold max |dz| of the native dz bit for bit
(a max does not depend on order); k is recomputed here from its exponent (math.frexp) and must equal the library's rule
(wunet_debug_train_dz_scale); the reference operand is built from that k. Block 0 stays fp32 and has no slot. The k range of
each run is printed.

In the runs of BN_REDUCTION the BatchNorm backward reductions of the middle block are also held to one fp32 ulp
(check_bn_reduction): its activation gradient is final after part 0 of the split backward, so a copy taken between the parts
is the exact input of train_bn_bwd_stats / train_bn_bwd_apply (train_bn_bwd_apply_amax at fp16_scaled), whose fp32
arithmetic is replayed from it.

A "blocks" run freezes the BatchNorm of some blocks, gives each block its own momentum, and leaves the gradient slots of the
lowest blocks null without asking for dx: below the lowest block that gets a gradient nothing may run, so those blocks' ga
(and fp16 scale slots) must still hold the NaN the workspace was filled with, and the reference stops its routing there.

The worst error/bar ratio of every quantity is printed per block, so the margins are on record (DESIGN §3)."""
import ctypes
import math
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import _lib

pytestmark = [pytest.mark.gpu]

ALL = ("fp32", "bf16", "tf32", "fp16_scaled")
# name -> shape, training precisions, BatchNorm modes ("batch" statistics / "frozen" running statistics / "blocks": the
# per-block settings below), and whether the backward computes parameter gradients (False: WUNET_TRAIN_NO_PARAM_GRADS, dx only)
CASES = {
    # the reference's own config/train (batch_size 120, sample_length 16384): fp32 weight gradient 4-52 tiles per CTA, bf16,
    # tf32 and fp16 14-233 items per CTA, BatchNorm reductions over ~2M samples per channel, dz of ~1e-7 in the upper blocks
    "production": dict(n=12, ci=24, B=120, T=16384, precisions=ALL, modes=("batch",), param_grads=(True,)),
    # L = 5 * 2^k: partial 128-position tiles (L = 320, 160), partial 64-position chunks (L = 160, 80), frames shorter than 64
    # samples, 5 -> 10 upsampling
    "odd_lengths": dict(n=12, ci=24, B=3, T=20480, precisions=ALL, modes=("batch", "frozen"), param_grads=(True,)),
    # channel counts that are not multiples of 8, 16, 32 or 64 (partial co / ci tiles of the weight-gradient kernels, padded
    # 32-channel K chunks of the tf32 forward)
    "channel_plan": dict(n=6, ci=20, B=5, T=2048, precisions=ALL, modes=("batch",), param_grads=(True,)),
    # a middle block with 32 x 1024 = 32768 values per channel (480 at the production shape) for the BatchNorm reductions, and
    # Cout = 8 blocks on the tensor-core kernels, whose tiles are mostly padding
    "long_middle": dict(n=4, ci=8, B=32, T=16384, precisions=ALL, modes=("batch",), param_grads=(True,)),
    # B = 1: BatchNorm over L only, two values per channel at the middle block
    "one_frame": dict(n=12, ci=24, B=1, T=8192, precisions=("fp32",), modes=("batch",), param_grads=(True,)),
    # L = 1 with B = 1 at the middle block, which eval-mode BatchNorm allows; with and without parameter gradients
    "one_value": dict(n=12, ci=24, B=1, T=4096, precisions=("fp32",), modes=("frozen",), param_grads=(True, False)),
    # the widest plan the training kernels accept at n = 12: Cin up to 1536 and Cout up to 768, 24 column tiles in the
    # input-gradient conv, ones / zeros read up to 1536 of their 2048 entries, a 1152-CTA fp32 weight-gradient grid (one
    # gridDim.z slice), 4-40 items per CTA on the tensor cores
    "wide_64": dict(n=12, ci=64, B=8, T=16384, precisions=ALL, modes=("batch",), param_grads=(True,)),
    # a wide plan at odd sizes: Cout = 8 (mod 16) at every odd multiple of 40, Cin not a multiple of 32 in the tf32 forward
    # chunks, partial 64- and 128-position tiles (T = 5 * 2^11), a middle block of L = 10
    "wide_40_odd": dict(n=10, ci=40, B=3, T=10240, precisions=ALL, modes=("batch", "frozen"), param_grads=(True,)),
    # fine-tuning with frozen layers (mode "blocks"): BatchNorm frozen on some blocks, each block its own momentum (1/3: a
    # cumulative average), the encoder's gradient slots null below block 6, block 7 with only the conv bias gradient, block 9
    # with only the BatchNorm parameter gradients, no dx: the backward stops early at block 6
    "mixed": dict(n=12, ci=24, B=4, T=4096, precisions=ALL, modes=("blocks",), param_grads=(True,),
                  bn_frozen=(0, 3, 12, 17, 24), momenta=tuple(1 / 3 if i == 5 else 0.02 * (i + 1) for i in range(25)),
                  slots={**{i: () for i in range(6)}, 7: ("b",), 9: ("gamma", "beta")}),
}
SLOTS = ("w", "b", "gamma", "beta")     # a block's gradient slots: conv weight, conv bias, BatchNorm weight, BatchNorm bias
# (case, precision) whose backward also runs as part 0 followed by part 1 (the data-parallel split) on a copy of the workspace
SPLIT = ({("production", "fp32"), ("odd_lengths", "bf16"), ("production", "tf32"), ("odd_lengths", "fp16_scaled"),
          ("wide_40_odd", "fp16_scaled"), ("wide_40_odd", "bf16")} | {("mixed", p) for p in ALL})
# runs (case, precision, mode, parameter gradients) whose middle block's BatchNorm backward is also replayed to one fp32 ulp
# from a copy of its activation gradient taken between part 0 and part 1; they run the split backward even if not in SPLIT
BN_REDUCTION = ([("production", p, "batch", True) for p in ("fp32", "bf16", "tf32")] +
                [("long_middle", p, "batch", True) for p in ("fp32", "bf16", "tf32")] +
                [("odd_lengths", p, "frozen", True) for p in ("fp32", "bf16", "tf32")] +
                [("production", "fp16_scaled", "batch", True), ("long_middle", "fp16_scaled", "batch", True),
                 ("odd_lengths", "fp16_scaled", "frozen", True)])

U32 = 2.0 ** -24                    # unit roundoff of fp32
U = 4 * U32                         # what the bars count per fp32 rounding of an elementwise formula: 4x its unit roundoff
FLIP = 2                            # weight of the bf16 rounding-flip allowance of interpolated operands (a bound: at most one flip)
EPS = float(np.float32(1e-5))       # kBnEps as the kernels see it
SLOPE = float(np.float32(0.1))      # kLreluSlope
MOMENTUM = 0.1
CONV_REL = 1e-5     # fp32 accumulation of <= 4320 products: worst case n u ~ 2.6e-4 of sum |products|
# weight gradients, a sum over B * L positions: fp32 FFMA chains of up to 52 x 128 positions per thread, then atomicAdd over
# the gridDim.z slices (measured <= 1e-6 of sum |products|); bf16 and tf32: wgmma's fp32 accumulation over up to 233 x 64
# positions per CTA (measured <= 9.4e-5 bf16, <= 3.4e-5 tf32 at the production shape, H100 80GB HBM3 at 700 W). Staging dz
# of the wrong tile moves outputs by 0.2-0.6 of sum |products|; tf32 operands truncated instead of rounded to nearest, by
# ~7e-4 at the production shape. fp16_scaled runs the bf16 MN-major kernel with the same items per CTA, and keeps its bar:
# worst err/bar 0.024 at the production shape and 0.16 over all cases (wide_64), where bf16 reaches 0.20 and tf32 0.26
# (both wide_40_odd), all on an H100 80GB HBM3 at 700 W.
WGRAD_REL = {"fp32": 1e-5, "bf16": 1e-3, "tf32": 3e-4, "fp16_scaled": 1e-3}
HEAD_REL = 1e-4     # 1x1 head gradients: fp32 products, warp sums, then one atomicAdd per warp over B * T / 32 warps
DOUBLE_REL = 1e-12  # double reductions of fp32 values: summation-order noise relative to the sum of magnitudes

RUNS = [(c, p, m, g) for c, d in CASES.items() for p in d["precisions"] for m in d["modes"] for g in d["param_grads"]]


def _run_id(r):
    c, p, m, g = r
    return f"{c}-{p}-{m}" + ("" if g else "-no_param_grads")


def make_pair(B, T, seed):
    g = np.random.Generator(np.random.PCG64(seed))
    clean = (0.1 * g.standard_normal((B, 1, T))).astype(np.float32)
    noisy = (clean + 0.05 * g.standard_normal((B, 1, T))).astype(np.float32)
    return noisy, clean


def ulp32(v):
    """Spacing of fp32 at |v| (float64 in, float64 out)."""
    a = v.abs().float()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def bf16r(v):
    """Round to bf16 (nearest even) the fp32 value the kernels hold, back in float64."""
    return v.float().bfloat16().double()


def tf32r(v):
    """cvt.rna.tf32.f32 of the fp32 value the kernels hold (round to nearest, ties away from zero: add half of the 13 dropped
    bits to the magnitude's bit pattern, then clear them), back in float64. On the tensor's device: the block tensors of the
    production case hold tens of millions of elements."""
    u = v.float().contiguous().view(torch.int32)
    return ((u + 0x1000) & -8192).view(torch.float32).double()


def f16r(v):
    """Round to fp16 (nearest even, subnormals kept, beyond +-65504 to +-inf: cvt.rn.f16.f32) the fp32 value the kernels hold,
    back in float64."""
    return v.float().half().double()


# operand rounding of a block's convolution kernels by the layout query's wgrad_tc: CUDA cores (none), bf16, tf32 or fp16
# tensor cores (fp16: the forward operands; dz is scaled first, see Step.dz_operand)
ROUND = {0: None, 1: bf16r, 2: tf32r, 3: f16r}


def dz_scale_exp(amax):
    """The k of fp16_scaled's dz scaling, restated: amax 2^k in [2^13, 2^14), 0 for 0 or a non-finite amax, clamped to +-126.
    frexp gives amax = m 2^e with m in [0.5, 1), so amax 2^k = m 2^(e + k) lies in [2^13, 2^14) for k = 14 - e."""
    if not (amax > 0 and math.isfinite(amax)):
        return 0
    return max(-126, min(126, 14 - math.frexp(amax)[1]))


def fma32(a, b, c):
    """fmaf(a, b, c) on fp32 tensors, exactly: a * b is exact in float64, TwoSum gives the error of the float64 sum, and a
    float64 sum that lands on the midpoint of two fp32 neighbours is resolved by the sign of that error."""
    p = a.double() * b.double()
    c = c.double()
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.float()
    rd = r.double()
    nb = torch.nextafter(r, torch.where(s > rd, torch.full_like(r, float("inf")), torch.full_like(r, float("-inf"))))
    nbd = nb.double()
    mid = (s != rd) & ((rd + nbd) * 0.5 == s)
    fix = mid & (e != 0) & ((e > 0) == (nbd > rd))
    return torch.where(fix, nb, r)


def bn_replay(z, mean, invstd, g, b):
    """The BatchNorm arithmetic of train_bn_act / train_bn_bwd_*: zh = fp32(fp32(z - mean) * invstd), y = fmaf(g, zh, b)."""
    c = lambda t: t[None, :, None].expand_as(z)          # noqa: E731
    zh = (z - c(mean)) * c(invstd)
    return zh, fma32(c(g), zh, c(b))


def upsample(p, L):
    """F.interpolate(scale_factor=2, mode="linear", align_corners=True) with the fp32 weights and indices of fetch_src:
    -> (float64 value of lam0 a + lam1 b, bound of the kernel's fp32 rounding of it, i0, i1, lam0, lam1)."""
    Lin = p.shape[-1]
    scale = np.float32(Lin - 1) / np.float32(L - 1) if L > 1 else np.float32(0)
    s = torch.tensor(scale, dtype=torch.float32, device=p.device) * torch.arange(L, dtype=torch.float32, device=p.device)
    i0 = s.long()
    i1 = torch.where(i0 < Lin - 1, i0 + 1, i0)
    lam1 = s - i0.float()
    lam0 = 1 - lam1
    t0 = lam0.double() * p[..., i0].double()
    t1 = lam1.double() * p[..., i1].double()
    return t0 + t1, 2.0 ** -23 * (t0.abs() + t1.abs()), i0, i1, lam0.double(), lam1.double()


def upsample_adjoint(d, Lin, i0, i1, lam0, lam1):
    out = torch.zeros(*d.shape[:-1], Lin, dtype=torch.float64, device=d.device)
    out.index_add_(-1, i0, d * lam0)
    out.index_add_(-1, i1, d * lam1)
    return out


class Report:
    """Worst |err| / bar (and worst |err|) per (block, quantity); failures are collected and asserted at the end."""

    def __init__(self, tag):
        self.tag, self.ratio, self.abs, self.fail, self.k = tag, {}, {}, [], {}    # k: fp16 dz scale exponent per block

    def check(self, blk, name, got, want, bar):
        err = (got.double() - want).abs()
        r = torch.where(err == 0, torch.zeros_like(err), err / bar)
        r = torch.nan_to_num(r, nan=float("inf"))
        worst = float(r.max()) if r.numel() else 0.0
        key = (blk, name)
        self.ratio[key] = max(self.ratio.get(key, 0.0), worst)
        self.abs[name] = max(self.abs.get(name, 0.0), float(torch.nan_to_num(err, nan=float("inf")).max()))
        if not worst <= 1.0:
            idx = np.unravel_index(int(r.argmax()), tuple(r.shape)) if r.dim() else ()
            self.fail.append(f"block {blk} {name}: err/bar {worst:.3g} at {idx}")

    def equal(self, blk, name, a, b):
        if not torch.equal(a, b):
            self.fail.append(f"block {blk} {name}: not bit-identical")

    def print(self):
        blocks = sorted({k[0] for k in self.ratio}, key=lambda b: (isinstance(b, str), b))
        for b in blocks:
            row = "  ".join(f"{n} {r:.1e}" for (bb, n), r in self.ratio.items() if bb == b)
            print(f"{self.tag} block {b}: {row}")
        per_q = {}
        for (_, n), r in self.ratio.items():
            per_q[n] = max(per_q.get(n, 0.0), r)
        print(f"{self.tag} worst err/bar: " + "  ".join(f"{n} {r:.2e}" for n, r in per_q.items()))
        print(f"{self.tag} worst |err|: " + "  ".join(f"{n} {e:.2e}" for n, e in self.abs.items()))
        if self.k:
            print(f"{self.tag} dz scale k: {min(self.k.values())} .. {max(self.k.values())} over blocks "
                  f"{min(self.k)} .. {max(self.k)} (" + " ".join(f"{b}:{k}" for b, k in sorted(self.k.items())) + ")")


class Step:
    """One native training step on a workspace of our own, with views of every block's tensors."""

    def __init__(self, case, prec, mode, param_grads):
        d = CASES[case]
        self.n, self.ci, self.B, self.T = n, ci, B, T = d["n"], d["ci"], d["B"], d["T"]
        self.prec, self.pgrads, self.blocks = prec, param_grads, mode == "blocks"
        self.nb = nb = 2 * n + 1
        # per block: BatchNorm on running statistics, the running-statistics factor as the kernels get it (fp32), and the
        # gradient slots the backward fills
        frozen = range(nb) if mode == "frozen" else d.get("bn_frozen", ())
        self.frozen = [i in frozen for i in range(nb)]
        self.momenta = [float(np.float32(d["momenta"][i] if self.blocks else MOMENTUM)) for i in range(nb)]
        self.slots = [d.get("slots", {}).get(i, SLOTS) if param_grads else () for i in range(nb)]
        # the lowest block that gets a gradient: a "blocks" run asks for no dx, so nothing below it runs (early stop)
        self.j = min(i for i in range(nb) if self.slots[i]) if self.blocks else 0
        dev = self.dev = torch.device("cuda:0")
        st = wo.make_state(n, ci, seed=21)
        plan = wo.channel_plan(n, ci)
        t = lambda k: torch.from_numpy(np.asarray(st[k])).to(dev).contiguous()   # noqa: E731
        self.w = [t(f"{p[0]}.0.weight") for p in plan]
        self.b = [t(f"{p[0]}.0.bias") for p in plan]
        self.gamma = [t(f"{p[0]}.1.weight") for p in plan]
        self.beta = [t(f"{p[0]}.1.bias") for p in plan]
        self.rm = [t(f"{p[0]}.1.running_mean") for p in plan]
        self.rv = [t(f"{p[0]}.1.running_var") for p in plan]
        self.rm0, self.rv0 = [v.clone() for v in self.rm], [v.clone() for v in self.rv]
        self.wo, self.bo = t("out.0.weight"), t("out.0.bias")
        noisy, clean = make_pair(B, T, 7)
        self.x = torch.from_numpy(noisy).to(dev)
        self.lay = [_lib.debug_train_layout(n, ci, B, T, i, prec) for i in range(self.nb)]
        self.lib = _lib.load()
        for i, lay in enumerate(self.lay):
            buf = (ctypes.c_longlong * 23)()                 # field 22: the fp16_scaled dz scale slot (-1: none)
            _lib.check(self.lib.wunet_debug_train_layout(n, ci, B, T, _lib.TRAIN_PRECISIONS[prec], i, buf, 23))
            lay["dz_slot"] = buf[22]
        self.k = {}                                         # fp16_scaled: block -> k of its dz scaling (check_backward)
        self.bn_frozen_arg = (ctypes.c_ubyte * nb)(*self.frozen)
        self.momenta_arg = (ctypes.c_float * nb)(*self.momenta)
        self.ctx = ctypes.c_void_p()
        _lib.check(self.lib.wunet_create(n, ci, 0, ctypes.byref(self.ctx)))
        nbytes = self.lib.wunet_train_workspace_bytes_prec(self.ctx, B, T, _lib.TRAIN_PRECISIONS[prec])
        assert nbytes == self.lay[0]["workspace_bytes"]
        self.ws = torch.full((nbytes // 4,), float("nan"), dtype=torch.float32, device=dev)   # unwritten reads show as NaN
        self.y = torch.full_like(self.x, float("nan"))
        self.flags = _lib.TRAIN_FROZEN_BN if mode == "frozen" else 0
        _lib.check(self.forward_rc())
        torch.cuda.synchronize()
        self.dy = (2.0 / self.y.numel()) * (self.y - torch.from_numpy(clean).to(dev))       # MSELoss(clean, y)'s gradient

    @staticmethod
    def ptrs(ts):
        """Device pointers of a list of tensors (None entries: null slots), or a null array for None."""
        return None if ts is None else (ctypes.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])

    def frozen_at(self, i):
        """Block i's BatchNorm normalises by (and keeps) its running statistics."""
        return self.frozen[i]

    def forward_rc(self):
        P = self.ptrs
        args = (self.ctx, self.x.data_ptr(), self.y.data_ptr(), self.B, self.T, P(self.w), P(self.b), P(self.gamma), P(self.beta),
                P(self.rm), P(self.rv), self.wo.data_ptr(), self.bo.data_ptr(), MOMENTUM, self.ws.data_ptr(), self.ws.numel() * 4,
                None, _lib.TRAIN_PRECISIONS[self.prec], self.flags)
        if self.blocks:
            return self.lib.wunet_train_forward_blocks(*args, self.bn_frozen_arg, self.momenta_arg)
        return self.lib.wunet_train_forward_ex(*args)

    def new_grads(self):
        """NaN-filled gradient buffers of the requested slots (None: a null slot), or None without parameter gradients."""
        if not self.pgrads:
            return None
        nan = lambda v: torch.full_like(v, float("nan"))                      # noqa: E731
        G = {k: [nan(v) if k in self.slots[i] else None for i, v in enumerate(src)]
             for k, src in zip(SLOTS, (self.w, self.b, self.gamma, self.beta))}
        return dict(G, wo=nan(self.wo), bo=nan(self.bo))

    def backward(self, ws, G, dx, part):
        P = self.ptrs
        flags = self.flags | (0 if self.pgrads else _lib.TRAIN_NO_PARAM_GRADS)
        g = G or {}
        args = (self.ctx, self.x.data_ptr(), self.y.data_ptr(), self.dy.data_ptr(), self.B, self.T, P(self.w), P(self.gamma),
                P(self.beta), self.wo.data_ptr(), P(g.get("w")), P(g.get("b")), P(g.get("gamma")), P(g.get("beta")),
                g["wo"].data_ptr() if G else None, g["bo"].data_ptr() if G else None, ws.data_ptr(), ws.numel() * 4, None,
                None if dx is None else dx.data_ptr(), part, _lib.TRAIN_PRECISIONS[self.prec], flags)
        if self.blocks:
            _lib.check(self.lib.wunet_train_backward_blocks(*args, self.bn_frozen_arg))
        else:
            _lib.check(self.lib.wunet_train_backward_ex(*args))

    def view(self, ws, i, field):
        d = self.lay[i]
        shape = (self.B, d["Cout"], d["L"]) if field in ("z", "act", "ga") else (d["Cout"],)
        o = d[field] // 4
        return ws[o:o + int(np.prod(shape))].view(shape)

    def scale_slot(self, ws, i):
        """fp16_scaled: block i's dz scale slot (one float: max |dz| of the block, written by the backward)."""
        o = self.lay[i]["dz_slot"] // 4
        return ws[o:o + 1]

    def dz_operand(self, i, dzd):
        """dz as block i's input- and weight-gradient kernels multiply it: rounded like the block's other operands, and at
        fp16_scaled f16(dz 2^k) 2^-k with the block's k (powers of two: exact in fp32 and float64)."""
        if self.lay[i]["wgrad_tc"] == 3:
            k = self.k[i]
            return f16r(dzd.float() * 2.0 ** k) * 2.0 ** -k
        return self.rounded(i, dzd)

    def rnd(self, i):
        """The operand rounding of block i's convolution kernels, or None (fp32 operands)."""
        return ROUND[self.lay[i]["wgrad_tc"]]

    def rounded(self, i, v):
        r = self.rnd(i)
        return v if r is None else r(v)

    def block_input(self, i):
        """-> (float64 block input as the block's kernels see it, rounding allowance of each operand or None, upsample data)."""
        d = self.lay[i]
        up = None
        if d["mode"] == 0:
            xin, xu = self.x.double(), None
        elif d["mode"] == 1:
            xin, xu = self.view(self.ws, i - 1, "act")[..., ::2].double(), None
        else:
            v, delta, *up = upsample(self.view(self.ws, i - 1, "act"), d["L"])
            skip = self.view(self.ws, 2 * self.n - i, "act").double()
            xin = torch.cat([v, skip], 1)
            xu = torch.cat([delta, torch.zeros_like(skip)], 1)
        r = self.rnd(i)
        if r is not None:
            if xu is not None:
                xu = r(xin + xu) - r(xin - xu)
            xin = r(xin)
        return xin, xu, up

    def weight(self, i):
        return self.rounded(i, self.w[i].double())


def check_forward(s, rep):
    n, B = s.n, s.B
    for i in range(s.nb):
        d = s.lay[i]
        pad = (d["ksize"] - 1) // 2
        z = s.view(s.ws, i, "z")
        xin, xu, _ = s.block_input(i)
        W = s.weight(i)
        want = F.conv1d(xin, W, s.b[i].double(), padding=pad)
        bar = CONV_REL * (F.conv1d(xin.abs(), W.abs(), padding=pad) + s.b[i].double().abs()[None, :, None])
        if xu is not None:
            bar += FLIP * F.conv1d(xu, W.abs(), padding=pad)
        rep.check(i, "z", z, want, bar)
        del xin, xu, want, bar
        mean, invstd = s.view(s.ws, i, "mean"), s.view(s.ws, i, "invstd")
        zd = z.double()
        if s.frozen_at(i):
            rep.equal(i, "mean", mean, s.rm0[i])
            inv = 1.0 / torch.sqrt(s.rv0[i].double() + EPS)
            rep.check(i, "invstd", invstd, inv, ulp32(inv))
            rep.equal(i, "running_mean", s.rm[i].view(torch.int32), s.rm0[i].view(torch.int32))     # bit-unchanged
            rep.equal(i, "running_var", s.rv[i].view(torch.int32), s.rv0[i].view(torch.int32))
        else:
            cnt = B * d["L"]
            mu = zd.mean((0, 2))
            var = ((zd - mu[None, :, None]) ** 2).mean((0, 2))
            inv = 1.0 / torch.sqrt(var + EPS)
            rep.check(i, "mean", mean, mu, ulp32(mu) + DOUBLE_REL * zd.abs().mean((0, 2)))
            rep.check(i, "invstd", invstd, inv, ulp32(inv))
            m = s.momenta[i]
            rm = (1 - m) * s.rm0[i].double() + m * mu
            rv = (1 - m) * s.rv0[i].double() + m * var * (cnt / (cnt - 1))
            rep.check(i, "running_mean", s.rm[i], rm, ulp32(rm) + DOUBLE_REL * zd.abs().mean((0, 2)))
            rep.check(i, "running_var", s.rv[i], rv, ulp32(rv))
        _, yv = bn_replay(z, mean, invstd, s.gamma[i], s.beta[i])
        act = torch.where(yv >= 0, yv, torch.tensor(SLOPE, dtype=torch.float32, device=s.dev) * yv)
        rep.check(i, "act", s.view(s.ws, i, "act"), act.double(), ulp32(act.double()))
        del z, zd, yv, act
    # head: y = tanh(sum_c Wo[c] a_last[c] + Wo[C] x + bo); fmaf chain of C + 1 terms, then tanhf (<= 2 ulp)
    a = s.view(s.ws, 2 * n, "act").double()
    wo = s.wo.view(-1).double()
    C = a.shape[1]
    pre = (wo[:C, None] * a).sum(1, keepdim=True) + wo[C] * s.x.double() + s.bo.double()
    mag = (wo[:C, None].abs() * a.abs()).sum(1, keepdim=True) + (wo[C] * s.x.double()).abs() + s.bo.double().abs()
    want = torch.tanh(pre)
    rep.check("head", "y", s.y, want, (C + 2) * U * mag + 6 * ulp32(want))


def check_backward(s, rep, wss, gsets, dxs):
    """wss / gsets / dxs: the workspaces, gradient sets and input gradients of one or more backward runs of the same forward;
    the first is checked in full, the others' dz slots, BatchNorm, bias and input gradients must equal it bit for bit and their
    atomically summed gradients (weights, head) pass the same bars. The routing stops at block s.j (the early stop of a
    "blocks" run): that block computes no input gradient, and the blocks below it must have been left untouched."""
    n, B, last = s.n, s.B, 2 * s.n
    ws = wss[0]
    if s.prec == "fp16_scaled" and (s.lay[0]["wgrad_tc"], s.lay[0]["dz_slot"]) != (0, -1):
        rep.fail.append(f"block 0: wgrad_tc {s.lay[0]['wgrad_tc']}, scale slot {s.lay[0]['dz_slot']} (fp32, no slot expected)")
    x = s.x.double()
    y = s.y.double()
    dy = s.dy.double()
    dpre = dy * (1 - y * y)
    e_dpre = 3 * U * dy.abs() * (1 + y * y)            # fp32 dy * (1 - y * y): three roundings
    wo = s.wo.view(-1).double()
    a_last = s.view(ws, last, "act").double()
    C = a_last.shape[1]
    if gsets[0] is not None:
        for G in gsets:
            gwo = G["wo"].view(-1)
            want = (dpre * a_last).sum((0, 2))
            bar = HEAD_REL * (dpre * a_last).abs().sum((0, 2)) + (e_dpre * a_last.abs()).sum((0, 2))
            rep.check("head", "g_out_w", gwo[:C], want, bar)
            rep.check("head", "g_out_w[x]", gwo[C], (dpre * x).sum(), HEAD_REL * (dpre * x).abs().sum() + (e_dpre * x.abs()).sum())
            rep.check("head", "g_out_b", G["bo"].view(()), dpre.sum(), HEAD_REL * dpre.abs().sum() + e_dpre.sum())
    pending = {last: (wo[:C, None] * dpre, wo[:C, None].abs() * e_dpre + U * (wo[:C, None] * dpre).abs())}
    del a_last
    G0 = gsets[0] or {k: [None] * s.nb for k in SLOTS}    # the requested gradient slots of block i: G0[slot][i] is not None
    for i in range(last, s.j - 1, -1):
        d = s.lay[i]
        pad = (d["ksize"] - 1) // 2
        da, e_da = pending.pop(i)
        z, mean, invstd = s.view(ws, i, "z"), s.view(ws, i, "mean"), s.view(ws, i, "invstd")
        zh32, yv = bn_replay(z, mean, invstd, s.gamma[i], s.beta[i])
        pos = yv >= 0
        del yv
        zh = zh32.double()
        del zh32
        dyv = torch.where(pos, da, SLOPE * da)
        e_dy = torch.where(pos, e_da, SLOPE * e_da) + U * dyv.abs()
        del pos, da, e_da
        isg = (invstd.double() * s.gamma[i].double())[None, :, None]
        cnt = B * d["L"]
        t1, t2 = dyv.sum((0, 2)), (dyv * zh).sum((0, 2))
        if s.frozen_at(i):
            want = isg * dyv
            bar = isg.abs() * e_dy + 4 * U * want.abs()
        else:
            s1, s2 = (t1 / cnt)[None, :, None], (t2 / cnt)[None, :, None]
            E1 = (e_dy.sum((0, 2)) / cnt)[None, :, None]
            E2 = ((e_dy * zh.abs()).sum((0, 2)) / cnt)[None, :, None]
            want = isg * (dyv - s1 - zh * s2)
            bar = isg.abs() * (e_dy + E1 + zh.abs() * E2) + 8 * U * isg.abs() * (dyv.abs() + s1.abs() + (zh * s2).abs())
            del s1, s2, E1, E2
        dz = s.view(ws, i, "ga")
        rep.check(i, "dz", dz, want, bar)
        del want, bar
        for w2 in wss[1:]:
            rep.equal(i, "dz (part split)", s.view(w2, i, "ga"), dz)
        if d["wgrad_tc"] == 3:
            # the scale slot holds max |dz| of this dz bit for bit; k is restated from it and checked against the library's rule
            amax = s.scale_slot(ws, i)
            rep.equal(i, "scale slot = max |dz|", amax, dz.abs().max().view(1))
            for w2 in wss[1:]:
                rep.equal(i, "scale slot (part split)", s.scale_slot(w2, i), amax)
            k = s.k[i] = rep.k[i] = dz_scale_exp(float(amax))
            if k != s.lib.wunet_debug_train_dz_scale(float(amax)):
                rep.fail.append(f"block {i} dz scale: k {k} restated, {s.lib.wunet_debug_train_dz_scale(float(amax))} by the library")
        if not s.frozen_at(i) or G0["gamma"][i] is not None or G0["beta"][i] is not None:
            # train_bn_bwd_stats ran: s1 = mean(dy), s2 = mean(dy zh), and the BatchNorm parameter gradients requested
            for name, t, e, mag in (("s1", t1, e_dy.sum((0, 2)), dyv.abs().sum((0, 2))),
                                    ("s2", t2, (e_dy * zh.abs()).sum((0, 2)), (dyv * zh).abs().sum((0, 2)))):
                rep.check(i, name, s.view(ws, i, name), t / cnt, (e + DOUBLE_REL * mag) / cnt + ulp32(t / cnt))
                gname, gkey = ("g_bn_bias", "beta") if name == "s1" else ("g_bn_weight", "gamma")
                if G0[gkey][i] is not None:
                    rep.check(i, gname, G0[gkey][i], t, e + DOUBLE_REL * mag + ulp32(t))
                    for G in gsets[1:]:
                        rep.equal(i, gname + " (part split)", G[gkey][i], G0[gkey][i])
        del dyv, e_dy, zh, t1, t2
        dzd = dz.double()
        if G0["b"][i] is not None:
            gb = dzd.sum((0, 2))
            rep.check(i, "g_conv_b", G0["b"][i], gb, ulp32(gb) + DOUBLE_REL * dzd.abs().sum((0, 2)))
            for G in gsets[1:]:
                rep.equal(i, "g_conv_b (part split)", G["b"][i], G0["b"][i])
        if G0["w"][i] is not None:
            xin, xu, _ = s.block_input(i)
            dzr = s.dz_operand(i, dzd)
            want = torch.nn.grad.conv1d_weight(xin, s.w[i].shape, dzr, padding=pad)
            bar = WGRAD_REL[s.prec] * torch.nn.grad.conv1d_weight(xin.abs(), s.w[i].shape, dzr.abs(), padding=pad)
            if xu is not None:
                bar += FLIP * torch.nn.grad.conv1d_weight(xu, s.w[i].shape, dzr.abs(), padding=pad)
            for G in gsets:
                rep.check(i, "g_conv_w", G["w"][i], want, bar)
            del xin, xu, dzr, want, bar
        if d["mode"] == 0:
            # dx = Wo[C] dy (1 - y^2) + the transposed block-0 convolution of dz0 (fp32 at both precisions)
            W = s.w[0].double()
            want = wo[C] * dpre + F.conv_transpose1d(dzd, W, padding=pad)
            bar = CONV_REL * (F.conv_transpose1d(dzd.abs(), W.abs(), padding=pad) + (wo[C] * dpre).abs()) + wo[C].abs() * e_dpre
            rep.check(0, "dx", dxs[0], want, bar)
            for dx2 in dxs[1:]:
                rep.equal(0, "dx (part split)", dx2, dxs[0])
            continue
        if i == s.j:
            break                                         # early stop: the lowest block that gets a gradient has no input gradient
        # input gradient of the block, routed to the producers of its input (decimation / interpolation + concat adjoints)
        W = s.weight(i)
        dzr = s.dz_operand(i, dzd)
        din = F.conv_transpose1d(dzr, W, padding=pad)
        e_din = CONV_REL * F.conv_transpose1d(dzr.abs(), W.abs(), padding=pad)
        del dzr, dzd
        if d["mode"] == 1:
            # g_prev[..., 2l] += din[..., l]: the skip gradient of an encoder is stored first, then this is added
            k = i - 1
            if k in pending:
                pa, pe = pending[k]
            else:
                Lk = s.lay[k]["L"]
                pa = torch.zeros(B, d["Cin"], Lk, dtype=torch.float64, device=s.dev)
                pe = torch.zeros_like(pa)
            pe[..., ::2] += e_din + U * (pa[..., ::2] + din).abs()
            pa[..., ::2] += din
            pending[k] = (pa, pe)
        else:
            c0 = d["Cin0"]
            if 2 * n - i >= s.j:                          # no skip gradient for an encoder below the early stop
                pending[2 * n - i] = (din[:, c0:].contiguous(), e_din[:, c0:].contiguous())
            _, _, up = s.block_input(i)
            Lin = d["L"] // 2
            ga = upsample_adjoint(din[:, :c0], Lin, *up)
            ge = upsample_adjoint(e_din[:, :c0] + 8 * U * din[:, :c0].abs(), Lin, *up)
            pending[i - 1] = (ga, ge)
        del din, e_din
    assert not pending
    # below the early stop nothing was issued: the activation gradients (and fp16 scale slots) still hold the workspace's NaN
    for i in range(s.j):
        for p, w in enumerate(wss):
            tag = "" if p == 0 else " (part split)"
            if not torch.isnan(s.view(w, i, "ga")).all():
                rep.fail.append(f"block {i} ga{tag}: written below the early stop at block {s.j}")
            if s.lay[i]["dz_slot"] >= 0 and not torch.isnan(s.scale_slot(w, i)).all():
                rep.fail.append(f"block {i} scale slot{tag}: written below the early stop at block {s.j}")


def check_bn_reduction(s, rep, ws, G, ga):
    """The BatchNorm backward of the middle block (n), replayed in the kernels' fp32 arithmetic from `ga`, a copy of its
    activation gradient taken between part 0 and part 1 (the exact input of train_bn_bwd_stats and train_bn_bwd_apply; ws and
    G are the workspace and gradients that run finished in). No error bar is inherited from the routed gradient:
    - s1 = mean(dy), s2 = mean(dy zh) and the parameter gradients g_bn_bias = sum dy, g_bn_weight = sum dy zh are double sums of
      fp32 terms (dy zh is exact in double), rounded once: 1 fp32 ulp + DOUBLE_REL of the sum of magnitudes. A float
      accumulator instead of a double one, or a dropped term, shows as many ulps.
    - dz = fp32(invstd gamma) * (dy - s1 - zh s2) from the native s1, s2 (zeros with frozen statistics): the kernel's formula,
      with zh s2 contracted into an FMA (the compiled train_bn_bwd_apply_kernel's FFMA; train_bn_bwd_apply_amax_kernel at
      fp16_scaled, the same formula), replayed exactly; 2 ulps."""
    i = s.n
    cnt = s.B * s.lay[i]["L"]
    z, mean, invstd = s.view(ws, i, "z"), s.view(ws, i, "mean"), s.view(ws, i, "invstd")
    zh, yv = bn_replay(z, mean, invstd, s.gamma[i], s.beta[i])
    dyv = torch.where(yv >= 0, ga, torch.tensor(SLOPE, dtype=torch.float32, device=s.dev) * ga)
    del yv
    d, zd = dyv.double(), zh.double()
    for name, terms, gname, gkey in (("s1", d, "g_bn_bias", "beta"), ("s2", d * zd, "g_bn_weight", "gamma")):
        t, mag = terms.sum((0, 2)), terms.abs().sum((0, 2))
        rep.check(i, name + " (1 ulp)", s.view(ws, i, name), t / cnt, ulp32(t / cnt) + DOUBLE_REL * mag / cnt)
        if G is not None:
            rep.check(i, gname + " (1 ulp)", G[gkey][i], t, ulp32(t) + DOUBLE_REL * mag)
        del terms
    del d, zd
    c = lambda t: t[None, :, None].expand_as(z)          # noqa: E731
    zeros = torch.zeros_like(mean)
    s1, s2 = (zeros, zeros) if s.frozen_at(i) else (s.view(ws, i, "s1"), s.view(ws, i, "s2"))
    want = (c(invstd) * c(s.gamma[i])) * fma32(-zh, c(s2), dyv - c(s1))
    rep.check(i, "dz (replay)", s.view(ws, i, "ga"), want.double(), 2 * ulp32(want.double()))


@pytest.mark.parametrize("run", RUNS, ids=[_run_id(r) for r in RUNS])
def test_training_kernels_block_by_block(run):
    case, prec, mode, pgrads = run
    t0 = time.perf_counter()
    s = Step(case, prec, mode, pgrads)
    bnred = run in BN_REDUCTION
    split = (case, prec) in SPLIT or bnred
    new_dx = lambda: None if s.blocks else torch.full_like(s.x, float("nan"))      # noqa: E731  (blocks runs: no dx)
    wss, gsets, dxs = [s.ws], [s.new_grads()], [new_dx()]
    if split:
        wss.append(s.ws.clone())                          # the backward turns ga into dz in place
        gsets.append(s.new_grads())
        dxs.append(new_dx())
    s.backward(wss[0], gsets[0], dxs[0], -1)
    if split:
        s.backward(wss[1], gsets[1], None, 0)
        ga_mid = s.view(wss[1], s.n, "ga").clone() if bnred else None     # final after part 0: the middle block feeds dec0 only
        s.backward(wss[1], gsets[1], dxs[1], 1)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    rep = Report(_run_id(run))
    with torch.no_grad():
        check_forward(s, rep)
        check_backward(s, rep, wss, gsets, dxs)
        if bnred:
            check_bn_reduction(s, rep, wss[1], gsets[1], ga_mid)
    torch.cuda.synchronize()
    _lib.load().wunet_destroy(s.ctx)
    rep.print()
    print(f"{_run_id(run)}: native step {t1 - t0:.1f} s (with set-up), float64 checks {time.perf_counter() - t1:.1f} s")
    assert not rep.fail, "\n".join(rep.fail[:40])


def test_one_value_per_channel_is_rejected_with_batch_statistics():
    """B = 1, T = 2^n_layers: the middle block sees one value per channel; torch.nn.BatchNorm1d raises in training mode, and
    so does the native forward (WUNET_EINVAL) unless BatchNorm uses the running statistics."""
    s = Step("one_value", "fp32", "frozen", True)          # the frozen forward accepts the shape
    s.flags = 0
    rc = s.forward_rc()
    assert rc == -1
    assert "Expected more than 1 value per channel when training" in _lib.load().wunet_last_error().decode()
    _lib.load().wunet_destroy(s.ctx)
