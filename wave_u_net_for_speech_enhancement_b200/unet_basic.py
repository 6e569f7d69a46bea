"""
Drop-in replacement for the reference's ``model/unet_basic.py`` (``Model``), forward path on H100.

Selected through the reference's own plugin loader (``util/utils.py:55-72``) by changing ONLY the
``"module"`` string of the ``"model"`` stanza (``config/train/train.json:22-26``)::

    "model": {"module": "wave_u_net_for_speech_enhancement_b200.unet_basic", "main": "Model", "args": {}}

Surface kept identical to the reference (SURVEY §8b):

* constructor ``Model(n_layers=12, channels_interval=24)``            (model/unet_basic.py:33)
* ``state_dict()``: the same 177 keys/shapes/dtypes, ``parameters()`` in the same registration
  order (conv.weight, conv.bias, bn.weight, bn.bias per block; encoder → middle → decoder → out), so
  reference checkpoints (``trainer/base_trainer.py:83-124``) and index-keyed Adam state interchange;
* ``forward(input[B,1,T]) -> [B,1,T]`` fp32, T a multiple of 2**n_layers   (model/unet_basic.py:77-100)

The sub-modules below exist ONLY as parameter/buffer containers with the reference's names; their
``forward`` is never called on the product path.  ``Model.forward`` hands device pointers to the
hand-written sm_90a kernels in ``libwunet_b200.so`` through the C ABI (``include/wunet_b200.h``).
There is no CPU or PyTorch fallback for the eval forward: a CPU tensor or a missing library raises.
"""
from __future__ import annotations

import ctypes
import threading
from typing import Dict, Optional, Tuple

import torch
import torch.nn as nn

from . import _lib

__all__ = ["Model", "DownSamplingLayer", "UpSamplingLayer"]


def _conv_bn_act(cin: int, cout: int, k: int, inplace: bool) -> nn.Sequential:
    # index 0 = Conv1d, 1 = BatchNorm1d, 2 = LeakyReLU  -> keys "<prefix>.0.weight", "<prefix>.1.running_mean", ...
    return nn.Sequential(
        nn.Conv1d(cin, cout, kernel_size=k, stride=1, padding=(k - 1) // 2),
        nn.BatchNorm1d(cout),
        nn.LeakyReLU(negative_slope=0.1, inplace=inplace),
    )


class DownSamplingLayer(nn.Module):
    """Parameter container named like the reference's encoder block (model/unet_basic.py:6-17)."""

    def __init__(self, channel_in: int, channel_out: int, kernel_size: int = 15):
        super().__init__()
        self.main = _conv_bn_act(channel_in, channel_out, kernel_size, inplace=False)

    def forward(self, ipt):  # pragma: no cover - only the opt-in torch training path calls this
        return self.main(ipt)


class UpSamplingLayer(nn.Module):
    """Parameter container named like the reference's decoder block (model/unet_basic.py:19-30)."""

    def __init__(self, channel_in: int, channel_out: int, kernel_size: int = 5):
        super().__init__()
        self.main = _conv_bn_act(channel_in, channel_out, kernel_size, inplace=True)

    def forward(self, ipt):  # pragma: no cover
        return self.main(ipt)


class _DeviceState:
    """Native context of one logical model on one CUDA device."""

    __slots__ = ("ctx", "weights_key", "workspaces", "last_ws")

    def __init__(self, ctx):
        self.ctx = ctx
        self.weights_key: Optional[Tuple] = None
        self.workspaces: Dict[Tuple, torch.Tensor] = {}
        self.last_ws: Optional[Tuple] = None


class _NativeState:
    """Registry of the native contexts (one per CUDA device) of ONE logical model.

    The Model holds it by reference and so does every shallow copy of the module: ``nn.DataParallel`` (what the unchanged
    ``trainer/base_trainer.py:26-27`` uses when several GPUs are visible) replicates with ``replica.__dict__ =
    self.__dict__.copy()``, so replicas SHARE this object, find the context of their device in it across forwards and never
    own (or destroy) one. ``copy.deepcopy`` / pickling give the copy a fresh, empty registry (``__reduce__``). The
    contexts are destroyed when the registry itself is collected, i.e. after the model and all its replicas are gone."""

    def __init__(self):
        self._lock = threading.Lock()
        self._dev: Dict[int, _DeviceState] = {}

    def __reduce__(self):
        # copy.deepcopy / pickle of the owning module: the copy gets its own, EMPTY registry (native handles are neither
        # copyable nor shareable between independent models)
        return (_NativeState, ())

    def device_state(self, idx: int, n_layers: int, channels_interval: int) -> _DeviceState:
        with self._lock:
            ds = self._dev.get(idx)
            if ds is None:
                ctx = ctypes.c_void_p()
                _lib.check(_lib.load().wunet_create(n_layers, channels_interval, idx, ctypes.byref(ctx)))
                ds = self._dev[idx] = _DeviceState(ctx)
            return ds

    def peek(self, idx: Optional[int] = None) -> Optional[_DeviceState]:
        with self._lock:
            if idx is None:
                return next(iter(self._dev.values()), None)
            return self._dev.get(idx)

    def invalidate_weights(self):
        with self._lock:
            for ds in self._dev.values():
                ds.weights_key = None

    def release(self):
        with self._lock:
            dev, self._dev = self._dev, {}
        for ds in dev.values():
            try:
                _lib.load().wunet_destroy(ds.ctx)
            except Exception:  # pragma: no cover - interpreter shutdown
                pass

    def __del__(self):
        try:
            self.release()
        except Exception:  # interpreter shutdown
            pass


class _NativeTrainStep(torch.autograd.Function):
    """forward = wunet_train_forward, backward = wunet_train_backward (include/wunet_b200.h). The activations live in a
    workspace tensor kept on the autograd context; parameter order: 4 per conv block (conv.weight, conv.bias, bn.weight,
    bn.bias) in forward order, then out.weight, out.bias."""

    @staticmethod
    def _ptr_array(tensors):
        return (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])

    @staticmethod
    def forward(ctx, model, x, *params):
        lib = _lib.load()
        blocks = model._blocks()
        nb = len(blocks)
        B, _, T = x.shape
        with torch.cuda.device(x.device):
            c = model._context(x.device)
            nbytes = lib.wunet_train_workspace_bytes(c, B, T)
            if nbytes == 0:
                _lib.check(-1)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
            y = torch.empty_like(x)
            conv_w = [params[4 * i] for i in range(nb)]
            conv_b = [params[4 * i + 1] for i in range(nb)]
            bn_w = [params[4 * i + 2] for i in range(nb)]
            bn_b = [params[4 * i + 3] for i in range(nb)]
            rmean = [blk[1].running_mean for blk in blocks]
            rvar = [blk[1].running_var for blk in blocks]
            momentum = float(blocks[0][1].momentum)
            stream = torch.cuda.current_stream(x.device).cuda_stream
            P = _NativeTrainStep._ptr_array
            _lib.check(lib.wunet_train_forward(c, x.data_ptr(), y.data_ptr(), B, T, P(conv_w), P(conv_b), P(bn_w), P(bn_b),
                                               P(rmean), P(rvar), params[-2].data_ptr(), params[-1].data_ptr(), momentum,
                                               ws.data_ptr(), ws.numel(), stream))
        ctx.model, ctx.ws, ctx.nb = model, ws, nb
        ctx.save_for_backward(x, y, *params)
        return y

    @staticmethod
    def backward(ctx, gy):
        from .train_step import GradientBucket, data_parallel_world
        lib = _lib.load()
        x, y, *params = ctx.saved_tensors
        nb = ctx.nb
        B, _, T = x.shape
        gy = gy.contiguous()
        # all gradients live in ONE flat buffer laid out in backward-completion order (train_step.GradientBucket); autograd
        # hands the views to .grad, so the all-reduce below needs no gather / scatter copies
        bucket = GradientBucket([p.shape for p in params], nb, x.device)
        grads = bucket.views
        reduce = ctx.model.data_parallel != "off" and data_parallel_world() > 1
        with torch.cuda.device(x.device):
            c = ctx.model._context(x.device)
            stream = torch.cuda.current_stream(x.device).cuda_stream
            P = _NativeTrainStep._ptr_array
            sel = lambda ts, k: [ts[4 * i + k] for i in range(nb)]          # noqa: E731
            for part in ((0, 1) if reduce else (-1,)):
                _lib.check(lib.wunet_train_backward_part(c, x.data_ptr(), y.data_ptr(), gy.data_ptr(), B, T, P(sel(params, 0)),
                                                         P(sel(params, 2)), P(sel(params, 3)), params[-2].data_ptr(),
                                                         P(sel(grads, 0)), P(sel(grads, 1)), P(sel(grads, 2)), P(sel(grads, 3)),
                                                         grads[-2].data_ptr(), grads[-1].data_ptr(), ctx.ws.data_ptr(),
                                                         ctx.ws.numel(), stream, part))
                if reduce:
                    # head + decoder gradients are final after part 0: their all-reduce overlaps part 1 (middle + encoders)
                    bucket.reduce_part(part)
            if reduce:
                bucket.finish()
        ctx.ws = None
        return (None, None, *grads)                          # no gradient for the model handle and for the input


class Model(nn.Module):
    """Wave-U-Net whose eval forward runs on hand-written sm_90a kernels.

    Extra keyword arguments (not in the reference; configs pass ``"args": {}`` so defaults apply):

    precision      "fp32_tc" (default): fp32-grade results on the tensor cores (bf16 hi + lo split, three MMAs per
                   product; <=1e-4 vs the reference, measured 1e-6; needs channels_interval % 8 == 0 and <= 32);
                   "fp32": the same contract on CUDA-core FFMA for any channel plan (slower);
                   "bf16": bf16 activations / operands on the tensor cores (the fastest path; ~6e-4 on the output).
    train_backend  "native" (default): a forward in training mode runs ``wunet_train_forward`` (BatchNorm with batch
                   statistics, running buffers updated) behind a ``torch.autograd.Function`` whose backward is
                   ``wunet_train_backward_part``; the reference's loss, ``loss.backward()`` and optimizer run unchanged
                   (trainer/trainer.py:34-38). fp32, checked against float64 golden steps.
                   "torch": opt-in composite of torch ops with the reference's semantics (runs on CPU too), used by the
                   CPU boundary tests that drive the unchanged ``trainer/trainer.py`` loop; not a measured hot path.
                   "none": a forward in training mode raises NotImplementedError.
    data_parallel  "auto" (default): when ``torch.distributed`` is initialised with more than one rank (one process per
                   GPU, SURVEY §8e) the native backward averages the gradients over the ranks — one flat bucket,
                   all-reduced in two parts so that the first overlaps the rest of the backward. "off": never.
    """

    def __init__(self, n_layers: int = 12, channels_interval: int = 24, precision: str = "fp32_tc",
                 train_backend: str = "native", data_parallel: str = "auto"):
        super().__init__()
        if precision not in _lib.PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(_lib.PRECISIONS)}, got {precision!r}")
        if train_backend not in ("none", "torch", "native"):
            raise ValueError("train_backend must be 'none', 'torch' or 'native'")
        self.n_layers = n_layers
        self.channels_interval = channels_interval
        if data_parallel not in ("auto", "off"):
            raise ValueError("data_parallel must be 'auto' or 'off'")
        self.precision = precision
        self.train_backend = train_backend
        self.data_parallel = data_parallel
        n, ci = n_layers, channels_interval

        enc_in = [1] + [i * ci for i in range(1, n)]
        enc_out = [(i + 1) * ci for i in range(n)]
        self.encoder = nn.ModuleList(DownSamplingLayer(a, b) for a, b in zip(enc_in, enc_out))
        self.middle = _conv_bn_act(n * ci, n * ci, 15, inplace=True)
        dec_out = enc_out[::-1]
        dec_in = [2 * n * ci] + [(2 * (n - j) + 1) * ci for j in range(1, n)]
        self.decoder = nn.ModuleList(UpSamplingLayer(a, b) for a, b in zip(dec_in, dec_out))
        self.out = nn.Sequential(nn.Conv1d(ci + 1, 1, kernel_size=1, stride=1), nn.Tanh())

        # native state (not part of state_dict); shared by reference with DataParallel replicas, see _NativeState
        self._native = _NativeState()

    # ------------------------------------------------------------------------------------------
    # native plumbing
    # ------------------------------------------------------------------------------------------
    def _blocks(self):
        return [e.main for e in self.encoder] + [self.middle] + [d.main for d in self.decoder]

    def _state(self, device: torch.device) -> _DeviceState:
        idx = device.index if device.index is not None else torch.cuda.current_device()
        return self._native.device_state(idx, self.n_layers, self.channels_interval)

    def _context(self, device: torch.device) -> ctypes.c_void_p:
        return self._state(device).ctx

    def _release(self):
        """Destroy the native contexts of this model (they are rebuilt lazily by the next forward)."""
        self._native.release()

    def _param_tensors(self):
        ts = []
        for blk in self._blocks():
            conv, bn = blk[0], blk[1]
            ts += [conv.weight, conv.bias, bn.weight, bn.bias, bn.running_mean, bn.running_var]
        ts += [self.out[0].weight, self.out[0].bias]
        return ts

    def _sync_weights(self, ctx, device: torch.device):
        """(Re)pack the library's weight copies when any parameter/buffer changed: optimizer.step()
        and load_state_dict bump ``_version``; .cpu()/.to() change ``data_ptr``."""
        ds = self._state(device)
        ts = self._param_tensors()
        key = tuple((t.data_ptr(), t._version) for t in ts)
        if key == ds.weights_key:
            return
        for t in ts:
            if t.device != device:
                raise RuntimeError(f"parameter on {t.device} but input on {device}: call model.to(device) first")
            if t.dtype != torch.float32 or not t.is_contiguous():
                raise RuntimeError("libwunet_b200 needs contiguous float32 parameters")
        nb = len(self._blocks())
        arrs = []
        for slot in range(6):
            arrs.append((ctypes.c_void_p * nb)(*[ts[6 * i + slot].data_ptr() for i in range(nb)]))
        stream = torch.cuda.current_stream(device).cuda_stream
        _lib.check(_lib.load().wunet_set_weights(ctx, *arrs, ts[-2].data_ptr(), ts[-1].data_ptr(), stream))
        ds.weights_key = key

    def _workspace(self, ctx, B: int, T: int, prec: int, device: torch.device) -> torch.Tensor:
        ds = self._state(device)
        key = (B, T, prec)
        ws = ds.workspaces.get(key)
        if ws is None:
            nbytes = _lib.load().wunet_workspace_bytes(ctx, B, T, prec)
            if nbytes == 0:
                _lib.check(-1)
            ds.workspaces = {}             # keep one shape resident (frames are fixed-length in practice)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
            ds.workspaces[key] = ws
        ds.last_ws = key
        return ws

    # ------------------------------------------------------------------------------------------
    # forward
    # ------------------------------------------------------------------------------------------
    def forward(self, input: torch.Tensor) -> torch.Tensor:  # noqa: A002 - reference argument name
        if self.training:
            if self.train_backend == "torch":
                return self._forward_torch_reference_semantics(input)
            if self.train_backend == "native":
                return self._forward_train_native(input)
            raise NotImplementedError(
                "this model was built with train_backend='none': call model.eval(), or construct it with "
                "train_backend='native' (default; sm_90a kernels) or 'torch' (composite PyTorch path).")
        # eval mode: like enhancement.py:66 (`model(chunk).detach().cpu()`, no torch.no_grad()) the result is
        # returned detached — the native path records no autograd graph.
        return self._forward_native(input)

    @property
    def reduces_gradients(self) -> bool:
        """True when ``loss.backward()`` through this model already averages the gradients over the data-parallel ranks."""
        from .train_step import data_parallel_world
        return (self.training and self.train_backend == "native" and self.data_parallel != "off"
                and data_parallel_world() > 1)

    def _forward_train_native(self, x: torch.Tensor) -> torch.Tensor:
        """Training-mode forward through libwunet_b200 (wunet_train_forward / wunet_train_backward behind a
        torch.autograd.Function): BatchNorm uses batch statistics and updates its running buffers, ``loss.backward()`` fills
        ``.grad`` of all 102 parameters, the caller's optimizer is used unchanged (trainer/trainer.py:34-38). fp32,
        correctness-first kernels (SURVEY §8f row N1)."""
        self._check_input(x)
        if not x.is_cuda:
            raise RuntimeError("wave_u_net_for_speech_enhancement_b200 has no CPU fallback: move the model and the "
                               "input to a CUDA (sm_90a) device")
        blocks = self._blocks()
        params = []
        for blk in blocks:
            params += [blk[0].weight, blk[0].bias, blk[1].weight, blk[1].bias]
        params += [self.out[0].weight, self.out[0].bias]
        for t in params:
            if t.device != x.device or t.dtype != torch.float32 or not t.is_contiguous():
                raise RuntimeError("libwunet_b200 needs contiguous float32 parameters on the input's device")
        y = _NativeTrainStep.apply(self, self._aligned(x), *params)
        for blk in blocks:                                   # torch.nn.BatchNorm1d bookkeeping (momentum is not None: unused)
            blk[1].num_batches_tracked += 1
        # the kernels updated running_mean / running_var through raw pointers (no _version bump): drop the folded copies
        self._native.invalidate_weights()
        return y

    def _check_input(self, x: torch.Tensor):
        if x.dim() != 3 or x.size(1) != 1:
            raise RuntimeError(f"expected input of shape [B, 1, T], got {tuple(x.shape)}")
        if x.dtype != torch.float32:
            raise RuntimeError(f"expected float32 input, got {x.dtype}")

    @staticmethod
    def _aligned(x: torch.Tensor) -> torch.Tensor:
        """contiguous and 16-byte aligned (the kernels use 128-bit loads; a slice ``wave[:, :, off:off+T]`` of a B=1 tensor
        is contiguous but only 4-byte aligned when ``off % 4 != 0``)"""
        x = x.contiguous()
        return x if x.data_ptr() % 16 == 0 else x.clone(memory_format=torch.contiguous_format)

    def _empty_batch(self, x: torch.Tensor) -> Optional[torch.Tensor]:
        """A batch of zero frames: the reference's eval forward returns an empty [0, 1, T] tensor (every layer accepts an empty
        batch) and still raises from torch.cat for a bad length; nothing to launch here."""
        if x.shape[0] != 0:
            return None
        T = int(x.shape[-1])
        if T < 1 or T % (1 << self.n_layers) != 0:
            raise _lib.WunetError(f"input length T={T} is not a multiple of 2^n_layers={1 << self.n_layers} (the reference raises "
                             "from torch.cat, model/unet_basic.py:95)")
        return torch.empty_like(x)

    def _forward_native(self, x: torch.Tensor) -> torch.Tensor:
        self._check_input(x)
        empty = self._empty_batch(x)
        if empty is not None:
            return empty
        if not x.is_cuda:
            raise RuntimeError("wave_u_net_for_speech_enhancement_b200 has no CPU fallback: move the model and the "
                               "input to a CUDA (sm_90a) device")
        x = self._aligned(x)
        B, _, T = x.shape
        lib = _lib.load()
        with torch.cuda.device(x.device):
            ctx = self._context(x.device)
            self._sync_weights(ctx, x.device)
            prec = _lib.PRECISIONS[self.precision]
            ws = self._workspace(ctx, B, T, prec, x.device)
            y = torch.empty_like(x)
            stream = torch.cuda.current_stream(x.device).cuda_stream
            _lib.check(lib.wunet_forward(ctx, x.data_ptr(), y.data_ptr(), B, T, prec, ws.data_ptr(), ws.numel(), stream))
        return y

    @torch.no_grad()
    def forward_host(self, x_host: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """End-to-end form of enhancement.py:64-66 (``model(chunk).detach().cpu()``): host tensor in,
        host tensor out; H2D copy, kernels and D2H copy are enqueued by ``wunet_forward_host``.
        Parameters must already live on a CUDA device. Pinned tensors give full copy bandwidth."""
        self._check_input(x_host)
        if x_host.is_cuda:
            raise RuntimeError("forward_host takes a host tensor")
        if self.training:
            raise NotImplementedError("forward_host is eval-only")
        empty = self._empty_batch(x_host)
        if empty is not None:
            return empty if out is None else out
        x_host = x_host.contiguous()
        device = self.out[0].weight.device
        if device.type != "cuda":
            raise RuntimeError("no CPU fallback: move the model to a CUDA device first")
        B, _, T = x_host.shape
        if out is None:
            out = torch.empty_like(x_host, pin_memory=x_host.is_pinned())
        with torch.cuda.device(device):
            ctx = self._context(device)
            cur = torch.cuda.current_stream(device)
            self._sync_weights(ctx, device)
            cur.synchronize()                      # packing ran on torch's stream; forward_host uses its own
            _lib.check(_lib.load().wunet_forward_host(ctx, x_host.data_ptr(), out.data_ptr(), B, T,
                                                      _lib.PRECISIONS[self.precision]))
        return out

    @torch.no_grad()
    def forward_host_stream(self, batches, outs=None):
        """Streaming form of :meth:`forward_host` for many host batches (every chunk of every clip, enhancement.py:49-74):
        yields one output tensor per input batch, in order; H2D copy, kernels and D2H copy of consecutive batches overlap
        (two batches in flight). ``batches``: iterable of pinned ``[B,1,T]`` float32 host tensors that must stay alive until
        their result has been yielded; ``outs``: optional iterable of pinned output tensors."""
        if self.training:
            raise NotImplementedError("forward_host_stream is eval-only")
        device = self.out[0].weight.device
        if device.type != "cuda":
            raise RuntimeError("no CPU fallback: move the model to a CUDA device first")
        lib = _lib.load()
        prec = _lib.PRECISIONS[self.precision]
        outs_it = iter(outs) if outs is not None else None
        pending = []                                   # (ticket, x, out)
        with torch.cuda.device(device):
            ctx = self._context(device)
            self._sync_weights(ctx, device)
            torch.cuda.current_stream(device).synchronize()        # packing ran on torch's stream
            for x in batches:
                self._check_input(x)
                if x.is_cuda:
                    raise RuntimeError("forward_host_stream takes host tensors")
                x = x.contiguous()
                out = next(outs_it) if outs_it is not None else torch.empty_like(x, pin_memory=x.is_pinned())
                B, _, T = x.shape
                ticket = ctypes.c_int(0)
                _lib.check(lib.wunet_stream_submit(ctx, x.data_ptr(), out.data_ptr(), B, T, prec, ctypes.byref(ticket)))
                pending.append((ticket.value, x, out))
                if len(pending) == 2:
                    t, _x, o = pending.pop(0)
                    _lib.check(lib.wunet_stream_wait(ctx, t))
                    yield o
            while pending:
                t, _x, o = pending.pop(0)
                _lib.check(lib.wunet_stream_wait(ctx, t))
                yield o

    @torch.no_grad()
    def read_level(self, block: int, B: int, T: int) -> torch.Tensor:
        """Diagnostic: full-resolution output of block ``block`` (0..2n: encoder i / middle / decoder j)
        of the LAST native forward with this (B, T), as fp32 [B, Cout, L] — what a forward hook on the
        reference's encoder[i] / middle / decoder[j] returns. Used by the per-level parity tests."""
        prec = _lib.PRECISIONS[self.precision]
        device = self.out[0].weight.device
        ds = self._native.peek(device.index if device.type == "cuda" else None)
        key = (B, T, prec)
        if ds is None or key not in ds.workspaces:
            raise RuntimeError("read_level: run a native forward with this (B, T) first")
        n = self.n_layers
        cout = self._blocks()[block][0].out_channels
        L = (T >> block) if block <= n else (T >> (2 * n - block))
        out = torch.empty(B, cout, L, dtype=torch.float32, device=device)
        ws = ds.workspaces[key]
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            _lib.check(_lib.load().wunet_read_level(ds.ctx, block, ws.data_ptr(), B, T, prec, out.data_ptr(), stream))
        return out

    def profile(self, enable: bool) -> None:
        """Measurement hook: record per-block CUDA events in subsequent native forwards."""
        ds = self._native.peek()
        if ds is None:
            raise RuntimeError("profile(): run a native forward first")
        _lib.check(_lib.load().wunet_profile_enable(ds.ctx, 1 if enable else 0))

    def profile_read(self):
        """Per-block device times (ms) of the last profiled forward: 2n+1 conv blocks, then the head."""
        cap = 2 * self.n_layers + 2
        buf = (ctypes.c_float * cap)()
        cnt = ctypes.c_int(0)
        _lib.check(_lib.load().wunet_profile_read(self._native.peek().ctx, buf, cap, ctypes.byref(cnt)))
        return [float(buf[i]) for i in range(cnt.value)]

    def last_launch_count(self) -> int:
        ds = self._native.peek()
        return 0 if ds is None else int(_lib.load().wunet_last_launch_count(ds.ctx))

    # ------------------------------------------------------------------------------------------
    # opt-in composite path with the reference's training semantics (NOT the product hot path)
    # ------------------------------------------------------------------------------------------
    def _forward_torch_reference_semantics(self, x: torch.Tensor) -> torch.Tensor:
        import torch.nn.functional as F
        skips = []
        o = x
        for layer in self.encoder:
            o = layer(o)
            skips.append(o)
            o = o[:, :, ::2]
        o = self.middle(o)
        for j, layer in enumerate(self.decoder):
            o = F.interpolate(o, scale_factor=2, mode="linear", align_corners=True)
            o = layer(torch.cat([o, skips[self.n_layers - 1 - j]], dim=1))
        return self.out(torch.cat([o, x], dim=1))

    # nn.Module hooks: any structural move invalidates the native context lazily (keys are checked per call)
    def _apply(self, fn, *args, **kwargs):
        r = super()._apply(fn, *args, **kwargs)
        self._native.invalidate_weights()
        return r
