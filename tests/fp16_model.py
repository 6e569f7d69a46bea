"""The arithmetic of the fp16 tensor-core path (Model(precision="fp16"), csrc/wunet_tc_f16.cu) restated on the CPU: the bf16
path's model (oracle/wunet_bf16_model.py) with every bf16 rounding replaced by the fp16 one the kernels use.

fp16 rounding (``f16``): saturate to +-65504, then round to nearest even, subnormals kept; a wide (float64) value is rounded
once, straight to fp16 (through fp32 first would round twice and can flip a tie). The packed interpolation of the decoder
producers (levels of at least 128 samples) computes d = f16(b - a) and r = f16(fma(lam, d, a)) in HFMA2 arithmetic, which does
not saturate: there ``f16_inf`` (round to nearest even, overflow -> inf) is the rounding."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle.wunet_bf16_model import _fold
from oracle.wunet_oracle import LRELU_SLOPE, channel_plan

F16_MAX = 65504.0


def f16_inf(t: torch.Tensor) -> torch.Tensor:
    """round to nearest even fp16 (numpy's conversion rounds float64 / float32 once), overflow -> inf; back as float32"""
    a = t.detach().cpu().numpy()
    with np.errstate(over="ignore"):
        return torch.from_numpy(a.astype(np.float16).astype(np.float32))


def f16(t: torch.Tensor) -> torch.Tensor:
    """saturating fp16 rounding of the kernels' stores (cvt.rn.satfinite.f16x2.f32)"""
    return f16_inf(t.clamp(-F16_MAX, F16_MAX))


def _block(x, st, prefix, k, quantise):
    w = torch.from_numpy(np.asarray(st[f"{prefix}.0.weight"], np.float32))
    if quantise:
        w = f16(w)
    acc = F.conv1d(x.double(), w.double(), None, padding=(k - 1) // 2).float()
    s, shift = _fold(st, prefix)
    v = acc * s[None, :, None] + shift[None, :, None]
    return torch.where(v >= 0, v, np.float32(LRELU_SLOPE) * v)


def _upsample_hfma2(prev):
    Lin = prev.shape[2]
    L = 2 * Lin
    up_scale = np.float32(Lin - 1) / np.float32(L - 1)
    l = torch.arange(L)
    m0 = torch.div(l - 1, 2, rounding_mode="floor")
    a = prev[:, :, m0.clamp(0, Lin - 1)].double()
    b = prev[:, :, (m0 + 1).clamp(0, Lin - 1)].double()
    lam = f16((l.double() * float(up_scale) - m0.double()).float()).double()     # fma in fp32, then fp16
    d = f16_inf(b - a).double()                                                    # exact difference, one rounding
    return f16_inf(lam[None, None, :] * d + a)                                     # fused: one rounding


def _block_folded(prev, skip, st, prefix):
    w = torch.from_numpy(np.asarray(st[f"{prefix}.0.weight"], np.float32))
    Cprev, Lin = prev.shape[1], prev.shape[2]
    L = 2 * Lin
    up_scale = np.float32(Lin - 1) / np.float32(L - 1) if L > 1 else np.float32(0)
    sidx = torch.arange(L, dtype=torch.float32) * up_scale
    i0 = sidx.to(torch.int64)
    i1 = i0 + (i0 < Lin - 1).to(torch.int64)
    lam1 = (sidx - i0.to(torch.float32)).double()
    U = torch.zeros(L, Lin, dtype=torch.float64)
    U[torch.arange(L), i0] += 1.0 - lam1
    U[torch.arange(L), i1] += lam1
    wp = w[:, :Cprev, :].double()
    weff = torch.zeros(w.shape[0], Cprev, L, Lin, dtype=torch.float64)
    for t in range(5):
        for l in range(L):
            lp = l + t - 2
            if 0 <= lp < L:
                weff[:, :, l, :] += wp[:, :, t, None] * U[lp][None, None, :]
    weff = f16(weff.float()).double()                      # expand_gemm_weights_kernel sums in fp32, then stores fp16
    acc = torch.einsum("bim,oilm->bol", prev.double(), weff)
    acc = acc + F.conv1d(skip.double(), f16(w[:, Cprev:, :]).double(), None, padding=2)
    s, shift = _fold(st, prefix)
    v = acc.float() * s[None, :, None] + shift[None, :, None]
    return torch.where(v >= 0, v, np.float32(LRELU_SLOPE) * v)


def _upsample_fp32(prev):
    Lin = prev.shape[2]
    L = 2 * Lin
    up_scale = np.float32(Lin - 1) / np.float32(L - 1) if L > 1 else np.float32(0)
    s = torch.arange(L, dtype=torch.float32) * up_scale
    i0 = s.to(torch.int64)
    i1 = i0 + (i0 < Lin - 1).to(torch.int64)
    lam1 = s - i0.to(torch.float32)
    lam0 = 1.0 - lam1
    return f16(lam0[None, None, :] * prev[:, :, i0] + lam1[None, None, :] * prev[:, :, i1])


def forward_fp16_model(state, x, n_layers=12, channels_interval=24, return_levels=False, forced=None, dense_bottom=None):
    """-> y [B,1,T] fp32 (and the fp16-valued outputs of the 2n+1 blocks as fp32 arrays; the last one unrounded). Arguments as
    oracle.wunet_bf16_model.forward_bf16_model (block 0 always on the CUDA cores: fp32 operands)."""
    plan = channel_plan(n_layers, channels_interval)
    n = n_layers
    xt = torch.from_numpy(np.asarray(x, np.float32))
    if dense_bottom is None:
        dense_bottom = xt.shape[0] >= 64
    levels, skips = [], []

    def keep(i, t):
        levels.append(t)
        return torch.from_numpy(np.asarray(forced[i], np.float32)) if (forced is not None and i < 2 * n) else t

    o = keep(0, f16(_block(xt, state, plan[0][0], 15, False)))
    skips.append(o)
    o = o[:, :, ::2]
    for i in range(1, n):
        o = keep(i, f16(_block(o, state, plan[i][0], 15, True)))
        skips.append(o)
        o = o[:, :, ::2]
    o = keep(n, f16(_block(o, state, "middle", 15, True)))
    for j in range(n):
        L = 2 * o.shape[2]
        if dense_bottom and L <= 16 and j != n - 1:
            v = _block_folded(o, skips[n - 1 - j], state, plan[n + 1 + j][0])
        else:
            up = _upsample_hfma2(o) if L >= 128 else _upsample_fp32(o)
            v = _block(torch.cat([up, skips[n - 1 - j]], dim=1), state, plan[n + 1 + j][0], 5, True)
        o = v if j == n - 1 else keep(n + 1 + j, f16(v))
        if j == n - 1:
            levels.append(o)
    w = torch.from_numpy(np.asarray(state["out.0.weight"], np.float32))[0, :, 0]
    b = np.float32(np.asarray(state["out.0.bias"], np.float32)[0])
    C = o.shape[1]
    pre = (o.double() * w[:C].double()[None, :, None]).sum(dim=1) + w[C].double() * xt[:, 0].double() + float(b)
    y = torch.tanh(pre).float()[:, None, :].numpy()
    return (y, [t.numpy() for t in levels]) if return_levels else y


def ulp_f16(v):
    """spacing of fp16 numbers at |v| (11 significant bits; 2^-24 in the subnormal range)"""
    return np.exp2(np.maximum(np.floor(np.log2(np.maximum(np.abs(v), 1e-30))), -14) - 10)
