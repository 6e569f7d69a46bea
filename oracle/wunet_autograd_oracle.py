"""
oracle/wunet_autograd_oracle.py — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The float64 training-step oracle of ``oracle/wunet_train_oracle.py`` extended to the rest of autograd through the reference
module (model/unet_basic.py:77-100):

* the gradient of the network INPUT (the head's raw-input channel, :98-99, plus the input gradient of encoder 0), which the
  training oracle computes internally and drops;
* BatchNorm1d in EVAL mode (frozen statistics): the forward normalises by running_mean / running_var and leaves them as they
  are; the backward has no mean terms, dz = invstd * gamma * LeakyReLU'(y) * da.

Written from the formulas, no autograd; the network wiring is the one of ``wunet_train_oracle.forward_train`` /
``backward``, which stay as they are. Pinned by ``tests/golden/autograd_*.npz`` (``oracle/gen_golden_autograd.py``: autograd
on the live reference module in float64, ``x.requires_grad_(True)``). Only ``tests/`` may import this module.
"""
from __future__ import annotations

from typing import Dict

import numpy as np

from . import wunet_train_oracle as wt
from .wunet_oracle import BN_EPS, LRELU_SLOPE, channel_plan


def _block_fwd_frozen(x, st, prefix, new_stats):
    """Conv1d -> BatchNorm1d (eval: running statistics) -> LeakyReLU; the running statistics are passed through unchanged."""
    w = st[f"{prefix}.0.weight"].astype(np.float64)
    b = st[f"{prefix}.0.bias"].astype(np.float64)
    g = st[f"{prefix}.1.weight"].astype(np.float64)
    be = st[f"{prefix}.1.bias"].astype(np.float64)
    rm = st[f"{prefix}.1.running_mean"].astype(np.float64)
    rv = st[f"{prefix}.1.running_var"].astype(np.float64)
    z = wt.conv1d_fwd(x, w, b)
    inv = 1.0 / np.sqrt(rv + BN_EPS)
    zh = (z - rm[None, :, None]) * inv[None, :, None]
    y = g[None, :, None] * zh + be[None, :, None]
    a = np.where(y >= 0, y, LRELU_SLOPE * y)
    new_stats[f"{prefix}.1.running_mean"] = rm
    new_stats[f"{prefix}.1.running_var"] = rv
    return a, (x, w, g, zh, inv, y)


def _block_bwd_frozen(da, cache, prefix, grads):
    """Gradient of the block input with frozen statistics (mean and invstd are constants); parameter gradients into `grads`."""
    x, w, g, zh, inv, y = cache
    dy = np.where(y >= 0, da, LRELU_SLOPE * da)
    grads[f"{prefix}.1.bias"] = dy.sum(axis=(0, 2))
    grads[f"{prefix}.1.weight"] = (dy * zh).sum(axis=(0, 2))
    dz = (inv * g)[None, :, None] * dy
    dx, dw, db = wt.conv1d_bwd(x, w, dz)
    grads[f"{prefix}.0.weight"] = dw
    grads[f"{prefix}.0.bias"] = db
    return dx


def forward(state: Dict[str, np.ndarray], x: np.ndarray, n_layers: int = 12, channels_interval: int = 24,
            frozen_bn: bool = False):
    """-> (y [B,1,T], running statistics after the step, cache). BatchNorm in training mode (batch statistics, running
    statistics updated as torch does), or with ``frozen_bn`` in eval mode (running statistics used and returned unchanged)."""
    plan = channel_plan(n_layers, channels_interval)
    n = n_layers
    block = _block_fwd_frozen if frozen_bn else wt._block_fwd
    x = x.astype(np.float64)
    new_stats: Dict[str, np.ndarray] = {}
    caches = []
    skips = []
    o = x
    for i in range(n):                                          # model/unet_basic.py:82-86
        o, c = block(o, state, plan[i][0], new_stats)
        caches.append(c)
        skips.append(o)
        o = o[:, :, ::2]
    o, c = block(o, state, plan[n][0], new_stats)              # :88
    caches.append(c)
    ups = []
    for j in range(n):                                          # :91-96
        U = wt.upsample_matrix(o.shape[2])
        ups.append((U, o.shape[1]))
        o = np.concatenate([np.einsum("bcm,lm->bcl", o, U, optimize=True), skips[n - 1 - j]], axis=1)
        o, c = block(o, state, plan[n + 1 + j][0], new_stats)
        caches.append(c)
    cat = np.concatenate([o, x], axis=1)                        # :98
    wo = state["out.0.weight"].astype(np.float64)
    bo = state["out.0.bias"].astype(np.float64)
    y = np.tanh(np.einsum("bcl,oc->bol", cat, wo[:, :, 0]) + bo[None, :, None])   # :99
    return y, new_stats, (caches, ups, cat, wo, y, n, plan, frozen_bn)


def backward(cache, dy: np.ndarray):
    """-> (parameter gradients, dx [B,1,T]) for the upstream gradient dy [B,1,T] of the output."""
    caches, ups, cat, wo, y, n, plan, frozen_bn = cache
    block = _block_bwd_frozen if frozen_bn else wt._block_bwd
    grads: Dict[str, np.ndarray] = {}
    dpre = dy * (1.0 - y * y)
    grads["out.0.weight"] = np.einsum("bol,bcl->oc", dpre, cat)[:, :, None]
    grads["out.0.bias"] = dpre.sum(axis=(0, 2))
    dcat = np.einsum("bol,oc->bcl", dpre, wo[:, :, 0])
    do = dcat[:, :-1]
    dx_head = dcat[:, -1:]                                      # the raw-input channel of the head
    dskips = [None] * n
    for j in reversed(range(n)):
        dcat_j = block(do, caches[n + 1 + j], plan[n + 1 + j][0], grads)
        U, cprev = ups[j]
        dskips[n - 1 - j] = dcat_j[:, cprev:]
        do = np.einsum("bcl,lm->bcm", dcat_j[:, :cprev], U, optimize=True)   # adjoint of the interpolation
    do = block(do, caches[n], plan[n][0], grads)
    for i in reversed(range(n)):
        da = dskips[i].copy()
        da[:, :, ::2] += do                                     # adjoint of o[:, :, ::2]
        do = block(da, caches[i], plan[i][0], grads)
    return grads, dx_head + do                                  # do: gradient of encoder 0's input


def mse_step(state, x: np.ndarray, clean: np.ndarray, n_layers: int = 12, channels_interval: int = 24,
             frozen_bn: bool = False):
    """One reference step up to the gradients with the input requiring grad: -> (loss, grads, running stats, y, dx)."""
    y, new_stats, cache = forward(state, x, n_layers, channels_interval, frozen_bn)
    diff = y - clean.astype(np.float64)
    loss = float((diff ** 2).mean())
    grads, dx = backward(cache, 2.0 * diff / diff.size)
    return loss, grads, new_stats, y, dx
