"""The arithmetic of the fp32_tc path (``Model(precision="fp32_tc")``, split precision on the tensor cores, DESIGN §5.2) and of
the fp32 CUDA-core path (``precision="fp32"``, DESIGN §5.3) restated in float64, block by block, with the error bars the
kernels' own arithmetic allows. Test infrastructure only.

Split values. Every fp32 value v the split path carries is a pair of bf16 halves, ``hi = bf16_rn(v)``, ``lo = bf16_rn(v - hi)``
(v - hi is exact in fp32): the epilogue of every block, the decoder producers and ``pack_tc_split_kernel`` (weights) compute
them so. ``read_level`` returns ``hi + lo``, which is exact in fp32; ``recover`` gets the halves back as ``hi = bf16_rn(r)``,
``lo = r - hi``. That is the stored pair except when |lo| is exactly half a bf16 ulp of hi: r then lies on a bf16 midpoint
and ties-to-even may pick the other hi (lo flips sign, hi + lo is unchanged). About 1 operand in 500 is such a tie. It only
moves the ``x_hi * w_lo`` product, by one bf16 ulp of x (<= 2^-7 |x|) times |w_lo| (<= 2^-8 |w|): at most 2^-15 of that
one product, which the block bar (1e-5 of the sum of all |products|) absorbs.

Blocks 1 .. 2n at fp32_tc. A product is ``x * w_hi + x_hi * w_lo`` with x = hi + lo (three MMAs: hi x w_hi, hi x w_lo,
lo x w_hi; the lo x w_lo term is dropped), the weights split with round-to-nearest-even. Encoders read the stored halves of
the decimated previous level. Decoders read the upsampled half as ``align_corners=True`` interpolation of the previous
level's stored hi + lo, rounded to fp32 and then split, and the skip half as its stored halves. The interpolation weights
are the producers' fp32 ones (the fp32 ``up_scale`` alone moves them by up to 5e-4 at l = 16383): the 8-row window of
full-length frames computes ``lam1 = fmaf(up_scale, l, -m0)``, the per-row path of packed frames (L < 128) and the fp32
path ``s = up_scale * l``, ``lam1 = s - (int)s``. The value ``lam0 a + lam1 b`` is then evaluated exactly and rounded once;
the kernels' fp32 evaluation of it is within an fp32 ulp, which moves a block by far less than its bar. The epilogue is
the folded scale / shift (``_fold``, fp32), ``fmaf``, LeakyReLU and the split store.

Block 0 at fp32_tc: fp32 samples and weights on the CUDA cores (``enc0_kernel_v2``, ``enc0_kernel``, ``enc0_wide_kernel``),
the same epilogue and split store. fp32 mode: every block as above with exact fp32 operands and an fp32 store.

Head (fused into the last block at fp32_tc, ``out_kernel`` at fp32): ``tanh(sum_c w_c a_c + w_C x + b)``. The fused head
reads the last block's unrounded fp32 activations; the model evaluates it on the stored hi + lo (``WUNET_TC_STORE_LAST=1``),
and the bar is widened by 2^-16 of sum |w_c a_c| for that storage.

Bars (``block_bar``, ``head_bar``), every quantity reported as error / bar:
- block value, fp32_tc: ``2^-16 (|got| + |model|) + ACC_REL |s| sum |products| + 4u |shift|``. Each side rounds its fp32
  value once to a split pair (|hi + lo - v| <= 2^-16 |v|); ACC_REL is the training step's z bar, the fp32 accumulation of the
  same wgmma K loops; the last term is the fp32 rounding of the folded shift, the floor of a block whose operands are all
  zero (the zero frame of ``edge_inputs``).
- block value, fp32: the same with 2 fp32 ulps of max(|got|, |model|) in place of the split term.
- LeakyReLU sign flips: the comparison is on activations, and LeakyReLU is 1-Lipschitz, so a pre-activation within the bar
  gives an activation within the same bar whichever sides of zero the two land on (a flip near zero costs (1 - 0.1) |v|,
  with |v| inside the accumulation bar).
- head: the training step's ``(C + 2) 4u`` of sum |terms| + 6 ulp, plus the storage widening above, plus ``TANH_FAST_ABS``
  at fp32_tc, whose head runs ``1 - 2 / (__expf(2 x) + 1)`` (few-ulp ``__expf`` and ``__fdividef``, absolute error ~1e-6)
  instead of ``tanhf``.

Mutations of one K chunk of one block (w_lo dropped for a chunk or for a decoder's skip chunks, lo data multiplied by w_lo,
the upsampled operand from hi only) move the block by 2-5e-4 of |s| sum |products|, 16-40x its bar at the worst element
(tests/test_split_model_cpu.py checks that the bars see each of them by at least 10x)."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from oracle.wunet_bf16_model import _fold
from oracle.wunet_oracle import LRELU_SLOPE, channel_plan

U32 = 2.0 ** -24              # unit roundoff of fp32
U = 4 * U32                   # per fp32 rounding of an elementwise formula, as the training step's bars count it
ACC_REL = 1e-5                # fp32 accumulation of the K loop, of |s| sum |products| (the training step's z bar)
SPLIT_REL = 2.0 ** -16        # |hi + lo - v| <= 2^-16 |v|: one rounding of an fp32 value to a split pair
TANH_FAST_ABS = 2.0 ** -19    # tanh_fast of the fused head (fp32_tc): __expf, __fdividef and 1 - q, absolute
PACKED_BELOW = 128            # split mode: levels shorter than this run packed tiles (the per-row producer path)
MODES = ("fp32_tc", "fp32")


def bf16_rn(t: torch.Tensor) -> torch.Tensor:
    """round-to-nearest-even bf16 of the fp32 value t holds (t: float32 or float64 holding an fp32 value), as float64"""
    return t.float().to(torch.bfloat16).double()


def f32(t: torch.Tensor) -> torch.Tensor:
    """one rounding to fp32, as float64"""
    return t.float().double()


def split(v: torch.Tensor):
    """-> (hi, lo) of fp32 values v: hi = bf16_rn(v), lo = bf16_rn(v - hi); both float64"""
    v = f32(v)
    hi = bf16_rn(v)
    return hi, bf16_rn(v - hi)


def recover(r: torch.Tensor):
    """-> (hi, lo) from a stored pair's sum r = hi + lo (exact in fp32): hi = bf16_rn(r), lo = r - hi. The stored pair up to
    the tie case of the module docstring."""
    r = f32(r)
    hi = bf16_rn(r)
    return hi, r - hi


def ulp32(v: torch.Tensor) -> torch.Tensor:
    """spacing of fp32 at |v|, float64"""
    a = v.abs().float()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def interp_weights(Lin: int, window: bool, device=None):
    """align_corners=True interpolation of Lin rows to 2 Lin, with the producers' fp32 weights -> (i0, i1, lam0, lam1).
    window: the 8-row window of full-length frames (rows (l-1)>>1 and that + 1, clamped; lam1 = fmaf(up_scale, l, -m0));
    else the per-row path of packed frames and the fp32 path's fetch_src (s = up_scale l, i0 = (int)s, lam1 = s - i0)."""
    L = 2 * Lin
    up = np.float32(Lin - 1) / np.float32(L - 1) if L > 1 else np.float32(0)
    l = np.arange(L)
    if window:
        m0 = (l - 1) >> 1
        lam1 = (float(up) * l - m0).astype(np.float32)          # exact in float64, one rounding: the fma
        i0, i1 = np.clip(m0, 0, Lin - 1), np.clip(m0 + 1, 0, Lin - 1)
    else:
        s = up * l.astype(np.float32)                           # fp32 product
        i0 = s.astype(np.int64)
        i1 = i0 + (i0 < Lin - 1)
        lam1 = s - i0.astype(np.float32)
    lam0 = np.float32(1) - lam1
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)      # noqa: E731
    return t(i0), t(i1), t(lam0.astype(np.float64)), t(lam1.astype(np.float64))


def upsample(prev: torch.Tensor, window: bool) -> torch.Tensor:
    """fp32 interpolation of prev [B, C, Lin] (float64 holding fp32 values) to [B, C, 2 Lin]: exact value, rounded once"""
    i0, i1, lam0, lam1 = interp_weights(prev.shape[2], window, prev.device)
    return f32(lam0 * prev[:, :, i0] + lam1 * prev[:, :, i1])


def weights(st, prefix: str, device=None) -> torch.Tensor:
    return torch.from_numpy(np.asarray(st[f"{prefix}.0.weight"], np.float32)).double().to(device)


def products(x: torch.Tensor, xh: torch.Tensor, w: torch.Tensor, mode: str, w_hi=None, w_lo=None):
    """-> (sum of products, sum of |products|) of a K-tap convolution, float64. fp32_tc: x (w_hi) + x_hi (w_lo); fp32: x w.
    w_hi / w_lo: the weight halves (default: split(w)); the sensitivity tests pass altered ones."""
    pad = (w.shape[2] - 1) // 2
    mag = F.conv1d(x.abs(), w.abs(), padding=pad)
    if mode == "fp32":
        return F.conv1d(x, w, padding=pad), mag
    if w_hi is None:
        w_hi, w_lo = split(w)
    return F.conv1d(x, w_hi, padding=pad) + F.conv1d(xh, w_lo, padding=pad), mag


def epilogue(acc: torch.Tensor, st, prefix: str, mode: str, store: bool = True):
    """fmaf(acc, s, shift), LeakyReLU, then the store: -> (stored value, unrounded fp32 activation, |s|, |shift|), each
    [B, C, L] / [1, C, 1] float64"""
    s, shift = _fold(st, prefix)
    s = s.double().to(acc.device)[None, :, None]
    shift = shift.double().to(acc.device)[None, :, None]
    v = f32(acc * s + shift)
    a = torch.where(v >= 0, v, f32(float(np.float32(LRELU_SLOPE)) * v))
    if not store or mode == "fp32":
        out = a
    else:
        hi, lo = split(a)
        out = hi + lo
    return out, a, s.abs(), shift.abs()


def stored(t: torch.Tensor, mode: str):
    """-> (x, x_hi) of a stored level (a read_level result): fp32_tc x = hi + lo; fp32 x and x_hi are the fp32 value"""
    if mode == "fp32":
        return t, t
    hi, lo = recover(t)
    return hi + lo, hi


def up_operand(prev: torch.Tensor, mode: str, hi_only: bool = False):
    """-> (x, x_hi) of a decoder's upsampled half from the previous level's stored values. fp32_tc: interpolate hi + lo in
    fp32 (``hi_only``: the hi halves alone, a sensitivity mutation), split, x = hi + lo of the split."""
    Lin = prev.shape[2]
    if mode == "fp32":
        u = upsample(prev, window=False)
        return u, u
    src = recover(prev)[0] if hi_only else prev
    u = upsample(src, window=2 * Lin >= PACKED_BELOW)
    hi, lo = split(u)
    return hi + lo, hi


@dataclass
class SplitModel:
    """Model of one forward: per block the stored value, the unrounded fp32 activation, |s| sum |products| and |shift|;
    the output and the head's sums of magnitudes."""
    levels: List[torch.Tensor] = field(default_factory=list)
    act: List[torch.Tensor] = field(default_factory=list)
    scale: List[torch.Tensor] = field(default_factory=list)
    shift: List[torch.Tensor] = field(default_factory=list)
    y: Optional[torch.Tensor] = None
    head_mag: Optional[torch.Tensor] = None        # sum |terms| of the head's pre-activation
    head_act_mag: Optional[torch.Tensor] = None    # sum_c |w_c a_c|: the part that reads the last block's activations


def block_input(levels, i: int, n: int, mode: str, xin: torch.Tensor, hi_only_up: bool = False):
    """-> (x, x_hi) operand of block i from the stored outputs of the blocks before it (levels[j], j < i) and the network
    input xin [B, 1, T] (block 0)"""
    if i == 0:
        return xin, xin
    if i <= n:
        return stored(levels[i - 1][:, :, ::2], mode)
    j = i - n - 1
    u, uh = up_operand(levels[i - 1], mode, hi_only_up)
    s, sh = stored(levels[n - 1 - j], mode)
    return torch.cat([u, s], 1), torch.cat([uh, sh], 1)


def forward_split_model(state, x, n_layers: int = 12, channels_interval: int = 24, mode: str = "fp32_tc", forced=None,
                        device=None) -> SplitModel:
    """Evaluate every block in float64 from the stored outputs of the blocks before it: the model's own (forced=None) or the
    GPU's (``forced``: the 2n or 2n + 1 read_level results, fp32 [B, C, L]; teacher forcing, so an error stays in its block).
    With 2n + 1 forced levels the head reads the GPU's stored last block. x: the network input [B, 1, T] as the kernels
    widen it (fp32, or the 16-bit samples widened exactly)."""
    assert mode in MODES, mode
    n = n_layers
    plan = channel_plan(n, channels_interval)
    tt = lambda a: (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.asarray(a, np.float32))).double().to(device)  # noqa: E731
    xin = tt(x)
    fz = None if forced is None else [tt(f) for f in forced]
    m = SplitModel()
    for i in range(2 * n + 1):
        prefix, _cin, _cout, _k = plan[i]
        xo, xh = block_input(m.levels if fz is None else fz, i, n, mode, xin)
        acc, mag = products(xo, xh, weights(state, prefix, device), "fp32" if i == 0 else mode)
        out, a, s, sh = epilogue(acc, state, prefix, mode)
        m.levels.append(out)
        m.act.append(a)
        m.scale.append(s * mag)
        m.shift.append(sh.expand_as(out))
        del xo, xh, acc, mag
    last = fz[2 * n] if fz is not None and len(fz) > 2 * n else m.levels[2 * n]
    w = torch.from_numpy(np.asarray(state["out.0.weight"], np.float32)).double().to(device)[0, :, 0]
    b = float(np.asarray(state["out.0.bias"], np.float32)[0])
    C = last.shape[1]
    terms = w[:C][None, :, None] * last
    pre = terms.sum(1, keepdim=True) + w[C] * xin + b
    m.head_act_mag = terms.abs().sum(1, keepdim=True)
    m.head_mag = m.head_act_mag + (w[C] * xin).abs() + abs(b)
    m.y = torch.tanh(pre)
    return m


def block_bar(got: torch.Tensor, model: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, mode: str) -> torch.Tensor:
    """the bar of a block value (module docstring), float64"""
    if mode == "fp32":
        store = 2 * ulp32(torch.maximum(got.abs(), model.abs()))
    else:
        store = SPLIT_REL * (got.abs() + model.abs())
    return store + ACC_REL * scale + U * shift


def head_bar(m: SplitModel, C: int, mode: str, y16: bool = False) -> torch.Tensor:
    """the bar of the output: the training step's head bar, the storage of the last block's activations (fp32_tc), the
    fused head's tanh_fast (fp32_tc) and, for a 16-bit output, its final rounding (half an ulp, at the larger side)"""
    bar = (C + 2) * U * m.head_mag + 6 * ulp32(m.y)
    if mode == "fp32_tc":
        bar = bar + SPLIT_REL * m.head_act_mag + TANH_FAST_ABS
    if y16:
        bar = bar + 0.5 * ulp_f16(m.y.abs() + bar)
    return bar


def ulp_f16(v: torch.Tensor) -> torch.Tensor:
    """spacing of fp16 numbers at |v| (11 significant bits; 2^-24 in the subnormal range)"""
    e = torch.floor(torch.log2(torch.clamp(v.abs(), min=1e-30)))
    return torch.exp2(torch.clamp(e, min=-14) - 10)


def ratio(err: torch.Tensor, bar: torch.Tensor) -> torch.Tensor:
    """err / bar, 0 where err is 0"""
    return torch.where(err == 0, torch.zeros_like(err), err / bar)
