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
* ``forward(input[B,1,T]) -> [B,1,T]`` fp32, T a multiple of 2**n_layers   (model/unet_basic.py:77-100); after
  ``model.half()`` / ``model.to(torch.bfloat16)`` the eval forward takes and returns that dtype, as the reference's modules do

The sub-modules below exist ONLY as parameter/buffer containers with the reference's names; their
``forward`` is never called on the product path.  ``Model.forward`` hands device pointers to the
hand-written sm_90a kernels in ``libwunet_b200.so`` through the C ABI (``include/wunet_b200.h``).
There is no CPU or PyTorch fallback for the eval forward: a CPU tensor or a missing library raises.
"""
from __future__ import annotations

import contextlib
import ctypes
import threading
from typing import Dict, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.modules import module as _nn_module
from torch.utils.hooks import RemovableHandle

from . import _lib

__all__ = ["Model", "DownSamplingLayer", "UpSamplingLayer"]

# element type of the eval forward's input and output -> WUNET_IO_* (a model whose parameters and buffers are all 16-bit runs
# with 16-bit input and output, widened / rounded at the two ends of the network)
_IO_DTYPES = {torch.float32: _lib.IO_F32, torch.float16: _lib.IO_F16, torch.bfloat16: _lib.IO_BF16}
_HALF = (torch.float16, torch.bfloat16)


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


def _native_call(lib, c, reducer, buf, call):
    """``call()`` (a training entry point, returning its status) with, when ``reducer`` is set, the BatchNorm all-reduce hook
    installed around it (wunet_train_set_bn_allreduce): the hook hands ``reducer`` the float64 view of ``buf`` the library
    names, to be summed over the ranks in place on the current stream. An exception raised in the reducer fails the call and
    is re-raised here; the hook is uninstalled in every case."""
    if reducer is None:
        _lib.check(call())
        return
    errors = []

    def hook(user, ptr, count, stream):
        try:
            off = (ptr - buf.data_ptr()) // buf.element_size()
            reducer(buf[off:off + count])
            return 0
        except BaseException as e:  # noqa: BLE001 - re-raised after the C call
            errors.append(e)
            return 1

    fn = _lib.BN_ALLREDUCE_FN(hook)                      # kept alive for the whole call
    _lib.check(lib.wunet_train_set_bn_allreduce(c, fn, None, buf.data_ptr(), buf.numel()))
    try:
        rc = call()
    finally:
        lib.wunet_train_set_bn_allreduce(c, _lib.BN_ALLREDUCE_FN(), None, None, 0)     # a null fn uninstalls
    if errors:
        raise errors[0]
    _lib.check(rc)


class _NativeTrainStep(torch.autograd.Function):
    """forward = wunet_train_forward_ex, backward = wunet_train_backward_ex (include/wunet_b200.h). The activations live in a
    workspace tensor kept on the autograd context; parameter order: 4 per conv block (conv.weight, conv.bias, bn.weight,
    bn.bias) in forward order, then out.weight, out.bias.

    ``blocks``: None (every BatchNorm in the mode ``flags`` says, one momentum, parameters all trainable or all frozen), or
    ``(bn_frozen, momenta)``, the per-block lists of a fine-tuning state: the step then runs wunet_train_forward_blocks /
    wunet_train_backward_blocks, and the backward computes only the gradients of the parameters that require grad (the
    others get None, and the gradient bucket holds only the trainable ones).

    ``flags``: 0 = BatchNorm with batch statistics, running buffers updated (.train()); ``_lib.TRAIN_FROZEN_BN`` = BatchNorm
    normalising by the running statistics, which stay untouched (.eval()); either may add ``_lib.TRAIN_DETERMINISTIC`` (weight
    and head gradients summed in a fixed order, with a larger workspace). The backward fills the gradient of ``x`` when it
    requires grad and those of the parameters when any of them does; with no parameter requiring grad it computes ``dx``
    only (no weight-gradient pass, no reduction, no all-reduce).

    ``reducer``: None, or the callable that sums a float64 CUDA view over the data-parallel ranks in place (nn.SyncBatchNorm):
    the forward's batch statistics and its backward's BatchNorm means then cover every rank's frames.

    ``export``: the blocks (forward order, 0 .. 2n) whose outputs the forward also returns, after ``y``, as fp32 [B, Cout, L]
    copies of the activations the workspace holds (what forward hooks on the block containers see). The gradients that reach
    them are added to those blocks' activation gradients inside the backward (wunet_train_backward_inject). Empty: the
    Function returns ``y`` alone and its backward makes exactly the calls it makes without hooks."""

    @staticmethod
    def _ptr_array(tensors):
        return (ctypes.c_void_p * len(tensors))(*[None if t is None else t.data_ptr() for t in tensors])

    @staticmethod
    def forward(ctx, model, flags, reducer, blocks_state, x, *params):
        return _NativeTrainStep._forward(ctx, model, flags, reducer, blocks_state, (), x, params)

    @staticmethod
    def _forward(ctx, model, flags, reducer, blocks_state, export, x, params):
        lib = _lib.load()
        blocks = model._blocks()
        nb = len(blocks)
        B, _, T = x.shape
        with torch.cuda.device(x.device):
            c = model._context(x.device)
            prec = _lib.TRAIN_PRECISIONS[model.train_precision]
            nbytes = lib.wunet_train_workspace_bytes_ex(c, B, T, prec, flags)
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
            stream = torch.cuda.current_stream(x.device).cuda_stream
            P = _NativeTrainStep._ptr_array
            # [sum dy | sum dy zhat | B L] of the widest block (n ci channels): the hook's exchange buffer
            bn_buf = None if reducer is None else torch.empty(2 * model.n_layers * model.channels_interval + 1,
                                                              dtype=torch.float64, device=x.device)
            args = (c, x.data_ptr(), y.data_ptr(), B, T, P(conv_w), P(conv_b), P(bn_w), P(bn_b), P(rmean), P(rvar),
                    params[-2].data_ptr(), params[-1].data_ptr())
            bn_frozen = None
            if blocks_state is None:
                momentum = next((float(blk[1].momentum) for blk in blocks if blk[1].momentum is not None), 0.1)
                _native_call(lib, c, reducer, bn_buf, lambda: lib.wunet_train_forward_ex(
                    *args, momentum, ws.data_ptr(), ws.numel(), stream, prec, flags))
            else:
                frozen, momenta = blocks_state
                bn_frozen = (ctypes.c_ubyte * nb)(*[1 if f else 0 for f in frozen])
                _native_call(lib, c, reducer, bn_buf, lambda: lib.wunet_train_forward_blocks(
                    *args, 0.0, ws.data_ptr(), ws.numel(), stream, prec, flags, bn_frozen, (ctypes.c_float * nb)(*momenta)))
            levels = []
            for i in export:                                 # copies of the activations, fp32 [B, Cout, L]
                lay = _lib.debug_train_layout(model.n_layers, model.channels_interval, B, T, i, model.train_precision)
                nel = B * lay["Cout"] * lay["L"]
                levels.append(ws[lay["act"]:lay["act"] + 4 * nel].view(torch.float32).view(B, lay["Cout"], lay["L"]).clone())
        # the backward runs at the precision, BatchNorm mode and synchronisation of ITS forward (and reads the bf16 weight
        # packings that forward left in ws)
        ctx.model, ctx.ws, ctx.nb, ctx.prec, ctx.flags = model, ws, nb, prec, flags
        ctx.reducer, ctx.bn_buf, ctx.bn_frozen, ctx.export = reducer, bn_buf, bn_frozen, export
        ctx.x_arg = 5 if export else 4                       # position of x among apply()'s arguments
        ctx.save_for_backward(x, y, *params)
        if not export:
            return y
        ctx.set_materialize_grads(False)                     # a level the loss does not use has no gradient to add
        return (y, *levels)

    @staticmethod
    def backward(ctx, gy, *g_levels):
        from .train_step import GradientBucket, data_parallel_world
        lib = _lib.load()
        x, y, *params = ctx.saved_tensors
        nb = ctx.nb
        B, _, T = x.shape
        gy = torch.zeros_like(y) if gy is None else gy.contiguous()
        g_act = [None] * nb                                  # upstream gradients of the exported block outputs
        for i, g in zip(ctx.export, g_levels):
            if g is not None:
                g_act[i] = g.float().contiguous()
        inject = any(g is not None for g in g_act)
        want_dx = ctx.needs_input_grad[ctx.x_arg]
        mask = ctx.needs_input_grad[ctx.x_arg + 1:]
        want_params = any(mask)
        per_block = ctx.bn_frozen is not None              # the forward ran wunet_train_forward_blocks
        dx = torch.empty_like(x) if want_dx else None
        flags = ctx.flags | (0 if want_params else _lib.TRAIN_NO_PARAM_GRADS)
        if want_params:
            # all gradients live in ONE flat buffer laid out in backward-completion order (train_step.GradientBucket); autograd
            # hands the views to .grad, so the all-reduce below needs no gather / scatter copies. Frozen parameters have no
            # slot (None: nothing is computed for them)
            bucket = GradientBucket([p.shape for p in params], nb, x.device, trainable=None if all(mask) else mask)
            grads = bucket.views
            reduce = ctx.model.data_parallel != "off" and data_parallel_world() > 1
        else:
            grads, reduce = [None] * len(params), False      # input gradient only: nothing to reduce (dx is per sample)
        with torch.cuda.device(x.device):
            c = ctx.model._context(x.device)
            stream = torch.cuda.current_stream(x.device).cuda_stream
            P = _NativeTrainStep._ptr_array
            sel = lambda ts, k: [ts[4 * i + k] for i in range(nb)]          # noqa: E731
            G = (lambda k: P(sel(grads, k))) if want_params else (lambda k: None)   # noqa: E731
            ptr = lambda t: None if t is None else t.data_ptr()               # noqa: E731
            for part in ((0, 1) if reduce else (-1,)):
                args = (c, x.data_ptr(), y.data_ptr(), gy.data_ptr(), B, T, P(sel(params, 0)), P(sel(params, 2)), P(sel(params, 3)),
                        params[-2].data_ptr(), G(0), G(1), G(2), G(3), ptr(grads[-2]), ptr(grads[-1]), ctx.ws.data_ptr(),
                        ctx.ws.numel(), stream)
                if inject:
                    # each block's hook gradient is added in the part that processes the block; dx goes to part 0 as well, as below
                    _native_call(lib, c, ctx.reducer, ctx.bn_buf, lambda: lib.wunet_train_backward_inject(
                        *args, ptr(dx), part, ctx.prec, flags, ctx.bn_frozen, P(g_act)))
                elif per_block:
                    # dx goes to part 0 as well: it tells the early stop that part 1 will need the gradient of block 0
                    _native_call(lib, c, ctx.reducer, ctx.bn_buf, lambda: lib.wunet_train_backward_blocks(
                        *args, ptr(dx), part, ctx.prec, flags, ctx.bn_frozen))
                else:
                    _native_call(lib, c, ctx.reducer, ctx.bn_buf, lambda: lib.wunet_train_backward_ex(
                        *args, ptr(dx) if part != 0 else None, part, ctx.prec, flags))
                if reduce:
                    # head + decoder gradients are final after part 0: their all-reduce overlaps part 1 (middle + encoders)
                    bucket.reduce_part(part)
            if reduce:
                bucket.finish()
        ctx.ws = ctx.bn_buf = ctx.reducer = ctx.bn_frozen = None
        # none for the model handle, the flags, the reducer, the block state (and the exported blocks)
        return (*[None] * ctx.x_arg, dx, *grads)


class _NativeTrainStepExport(_NativeTrainStep):
    """:class:`_NativeTrainStep` that also returns the outputs of the blocks ``export`` (a non-empty tuple), for forward hooks."""

    @staticmethod
    def forward(ctx, model, flags, reducer, blocks_state, export, x, *params):
        return _NativeTrainStep._forward(ctx, model, flags, reducer, blocks_state, export, x, params)


class Model(nn.Module):
    """Wave-U-Net whose eval forward runs on hand-written sm_90a kernels.

    Extra keyword arguments (not in the reference; configs pass ``"args": {}`` so defaults apply):

    precision      "fp32_tc" (default): fp32-grade results on the tensor cores (bf16 hi + lo split, three MMAs per
                   product; <=1e-4 vs the reference, measured 1e-6; needs channels_interval % 8 == 0 and <= 64);
                   "fp32": the same contract on CUDA-core FFMA for any channel plan (slower);
                   "bf16": bf16 activations / operands on the tensor cores (the fastest path; ~6e-4 on the output);
                   "fp16": the bf16 contract with fp16 activations / operands (11-bit significand, the precision of the
                   TF32 convolutions cuDNN runs for the reference on an H100) at bf16's speed. fp16 stores saturate at
                   +-65504; activations near that range are not what this model produces. Same channel-plan needs as
                   "fp32_tc". Inference only: ``train_precision`` does not accept it.
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
    train_precision  arithmetic of the native training step's three convolution-shaped passes (forward conv, input
                   gradient, weight gradient). "fp32" (default): fp32 FFMA. "bf16": mixed precision — their operands (block
                   input, weights, dz) are rounded to bf16 and the products accumulated in fp32 on the tensor cores; z,
                   BatchNorm, the head and all gradients stay fp32, parameters stay fp32 (the caller's optimizer is unchanged).
                   ``torch.autocast(bfloat16)`` semantics for Conv1d, except that z is kept in fp32. "tf32": the same with
                   the operands rounded to tf32 (11 significant bits, round to nearest) instead, which is what cuDNN does
                   for Conv1d on an H100 under PyTorch's default ``torch.backends.cudnn.allow_tf32 = True``, i.e. the
                   reference's own training arithmetic there (that flag does not select it: the default stays "fp32").
                   "fp16_scaled": the same with fp16 operands (round to nearest even) at bf16's speed, and each block's
                   dz scaled inside the library by 2^k chosen on the device (max |dz| 2^k in [2^13, 2^14)), its results
                   by 2^-k: exact, so no loss scaling is needed; non-finite values are not saturated and reach the
                   gradients (a ``torch.amp.GradScaler`` then skips the step). Plain "fp16" (unscaled, autocast semantics)
                   is not a training precision. "bf16", "tf32" and "fp16_scaled" only with train_backend="native". Not
                   part of the state_dict.
    eval_autograd  when an eval-mode forward records an autograd graph (grad mode on, train_backend "native" or "torch").
                   "input" (default): when the input requires grad — ``x.grad`` of an upstream model or front end, input
                   gradients of an adversarial perturbation. "always": also when some parameter requires grad, for
                   fine-tuning with frozen BatchNorm statistics (``model.eval()`` then ``loss.backward()``). "off": the eval
                   forward always returns a detached tensor. A recorded eval forward runs the native training kernels at
                   ``train_precision`` with BatchNorm normalising by the running statistics, which it leaves untouched (the
                   reference's eval-mode BatchNorm), and keeps the activations for the backward; gradients reach ``x`` and
                   every parameter that requires grad, averaged over data-parallel ranks like the training backward. Every
                   other eval forward takes the inference kernels (``precision``) and returns a detached tensor. "always" is
                   not the default because a caller that runs inference without ``torch.no_grad()`` (enhancement.py:66) would
                   then pay for the training kernels and their workspace on every call. Not part of the state_dict.

    Deterministic mode (no constructor argument): a native training-kernel forward (``.train()``, or an eval forward that
    records a graph) made while ``torch.backends.cudnn.deterministic`` or ``torch.are_deterministic_algorithms_enabled()``
    is on sums the weight and head gradients in an order fixed by the shapes instead of with float atomics, and its
    backward follows. The step is then bitwise repeatable (``y``, running buffers, every gradient, ``x.grad``) for the same
    state, input, ``train_precision`` and GPU model. This is how the reference's ``"cudnn_deterministic": true``
    (config/train/train.json, trainer/base_trainer.py:140-143) reaches the native step. It costs a scratch region in the
    training workspace (about 70 MB in fp32, 22 MB in bf16 at the reference's batch of 120 x 16384). Note that
    ``torch.use_deterministic_algorithms(True)`` also makes torch fill every ``torch.empty`` tensor, including the training
    workspace, on every step (``torch.utils.deterministic.fill_uninitialized_memory``); that setting is left to the caller.

    Synchronised BatchNorm (no constructor argument): after ``nn.SyncBatchNorm.convert_sync_batchnorm(model)`` a native
    training forward with batch statistics, and its backward, compute the BatchNorm statistics over every rank's frames when
    ``torch.distributed`` is initialised and the containers' process group has more than one rank, as ``nn.SyncBatchNorm``
    does (three small all-reduces per block, on the current stream). The running statistics then agree on every rank, and
    with equal shards the data-parallel step equals the single-process step on the concatenated batch.

    Fine-tuning with frozen layers (no constructor argument): the native step honours each BatchNorm container's own
    ``.training`` (batch statistics, or the running statistics left untouched), ``momentum`` (``None``: the cumulative
    factor ``1 / num_batches_tracked``) and ``num_batches_tracked``, and each parameter's ``requires_grad``: a frozen
    parameter gets no gradient and costs no weight-gradient pass or all-reduce, and the backward stops below the lowest block
    that still needs a gradient. So ``model.train()``, ``m.eval()`` on every ``nn.BatchNorm1d`` and
    ``model.encoder.requires_grad_(False)`` compute what the reference computes. An ``.eval()`` model with a container in
    ``.train()`` runs the training kernels (detached unless ``eval_autograd`` records a graph); ``forward_host`` and
    ``forward_host_stream`` refuse it. Not supported: BatchNorm with ``affine=False`` or ``track_running_stats=False``, or an
    ``eps`` other than the library's 1e-5.

    Half models (no constructor argument): after ``model.half()`` or ``model.to(torch.bfloat16)`` (every parameter and buffer
    of that one dtype) the eval forward, ``forward_host`` and ``forward_host_stream`` take an input of that dtype and return
    one, as the reference's modules do. The computation is that of the same ``precision`` on the float32 model with the
    parameters and samples widened to fp32 (exact), and the output rounded once to the 16-bit dtype (nearest even): so
    ``half_model(x16) == float_model(x16.float()).to(x16.dtype)`` bit for bit. A float32 input to a half model, a 16-bit
    input to a float32 model and mixed parameter dtypes raise RuntimeError. Training a half model (``.train()``, or an eval
    forward that records a graph) raises too: the native training step keeps float32 parameters, and ``train_precision``
    is how to train in 16 bits. ``read_level`` stays fp32.

    Forward hooks (no constructor argument): ``register_forward_hook`` (``with_kwargs`` and ``always_call`` included) on
    ``encoder[i]``, ``encoder[i].main``, ``middle``, ``decoder[j]``, ``decoder[j].main`` and ``out``, and global module forward
    hooks, fire from the native forward in the reference's order (encoder 0 .. n-1, middle, decoder 0 .. n-1, out; a block's
    ``main`` before the block) after its kernels are enqueued and before ``forward`` returns. A hook receives ``(module,
    (input,), output)`` with the reference's meaning: the block's full-resolution output [B, Cout, L] (an encoder's before
    decimation; ``out``: the model output), and as input x, the previous output ``[:, :, ::2]`` or, for a decoder block,
    ``cat([F.interpolate(prev, scale_factor=2, mode="linear", align_corners=True), skip])`` computed with torch from the
    exported outputs (torch's arithmetic). Outputs are fresh tensors of the model's dtype: at the inference precisions the block
    output the next block reads, widened to fp32 and, for a half model, rounded once; in the training kernels (``.train()``, or
    an eval forward that records a graph) fp32 copies of the activations that are extra outputs of the native autograd
    Function, so a loss on them (feature matching, deep supervision, distillation) back-propagates through the native backward.
    Refused, naming the module: a hook that returns a value (RuntimeError), forward pre-hooks and hooks on the Conv1d /
    BatchNorm1d / LeakyReLU / Tanh inside a block (NotImplementedError: the kernels fuse them), and module backward hooks on any
    sub-module (NotImplementedError). Changing a hook's output in place does not change the forward. Without hooks the forward
    makes exactly the calls it makes otherwise. ``forward_host``, ``forward_host_stream`` and ``enhance_waveforms`` do not go
    through ``forward`` and fire no hooks.
    """

    def __init__(self, n_layers: int = 12, channels_interval: int = 24, precision: str = "fp32_tc",
                 train_backend: str = "native", data_parallel: str = "auto", train_precision: str = "fp32",
                 eval_autograd: str = "input"):
        super().__init__()
        if precision not in _lib.PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(_lib.PRECISIONS)}, got {precision!r}")
        if train_backend not in ("none", "torch", "native"):
            raise ValueError("train_backend must be 'none', 'torch' or 'native'")
        self.n_layers = n_layers
        self.channels_interval = channels_interval
        if data_parallel not in ("auto", "off"):
            raise ValueError("data_parallel must be 'auto' or 'off'")
        if train_precision not in _lib.TRAIN_PRECISIONS:
            raise ValueError(f"train_precision must be one of {sorted(_lib.TRAIN_PRECISIONS)}, got {train_precision!r}")
        if train_precision != "fp32" and train_backend != "native":
            raise ValueError(f"train_precision={train_precision!r} needs train_backend='native' (got {train_backend!r})")
        if eval_autograd not in ("input", "always", "off"):
            raise ValueError(f"eval_autograd must be 'input', 'always' or 'off', got {eval_autograd!r}")
        self.precision = precision
        self.train_backend = train_backend
        self.data_parallel = data_parallel
        self.train_precision = train_precision
        self.eval_autograd = eval_autograd
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
        # private seam: a callable summing a float64 CUDA view over the ranks in place forces the synchronised BatchNorm path
        # (see _bn_sync_reducer)
        self._bn_allreduce = None
        # RemovableHandle.next_id at the last hook scan that found no hook (see _forward_hook_plan)
        self._hook_free_at = None

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

    def _param_dtype(self) -> Optional[torch.dtype]:
        """The dtype shared by every parameter and buffer the forward reads, or None when they differ."""
        dts = {t.dtype for t in self._param_tensors()}
        return dts.pop() if len(dts) == 1 else None

    def _sync_weights(self, ctx, device: torch.device):
        """(Re)pack the library's weight copies when any parameter/buffer changed: optimizer.step()
        and load_state_dict bump ``_version``; .cpu()/.to()/.half() change ``data_ptr``. 16-bit parameters (all of one
        dtype) are handed to the library as fp32 copies: widening is exact, and the library copies what it reads."""
        ds = self._state(device)
        ts = self._param_tensors()
        key = tuple((t.data_ptr(), t._version) for t in ts)
        if key == ds.weights_key:
            return
        dtype = self._param_dtype()
        for t in ts:
            if t.device != device:
                raise RuntimeError(f"parameter on {t.device} but input on {device}: call model.to(device) first")
            if dtype not in _IO_DTYPES or not t.is_contiguous():
                raise RuntimeError("libwunet_b200 needs contiguous float32 parameters, or all of them float16 or all bfloat16 "
                                   f"(got {', '.join(sorted({str(u.dtype) for u in ts}))})")
        if dtype != torch.float32:
            ts = [t.float() for t in ts]        # freed after the call: the packing kernels run on this stream first
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
        # eval mode: a forward that needs a graph (see eval_autograd: the input requires grad, or "always" and a parameter
        # does) runs the training kernels with eval-mode BatchNorm, or the composite path for train_backend="torch".
        # A BatchNorm container switched back to .train() needs batch statistics, which only the training kernels compute:
        # that forward takes them too, per-block modes, and returns a detached tensor unless it records a graph.
        # Everything else — enhancement.py:66 (`model(chunk).detach().cpu()`, no torch.no_grad()), validation under
        # torch.no_grad(), an empty batch — takes the inference kernels and gets a detached result.
        if input.numel() != 0:
            records = self._eval_records_graph(input)
            if self._bn_any_training():
                if self.train_backend == "none":
                    raise NotImplementedError(
                        "a BatchNorm container of this eval-mode model is in training mode, which needs the training kernels: "
                        "construct the model with train_backend='native' (default) or 'torch', or call .eval() on it")
                with contextlib.nullcontext() if records else torch.no_grad():
                    if self.train_backend == "native":
                        return self._forward_train_native(input)
                    return self._forward_torch_reference_semantics(input)
            if records:
                if self.train_backend == "native":
                    return self._forward_train_native(input)
                return self._forward_torch_reference_semantics(input)
        return self._forward_native(input)

    def _bn_any_training(self) -> bool:
        return any(blk[1].training for blk in self._blocks())

    def _eval_records_graph(self, x: torch.Tensor) -> bool:
        if self.eval_autograd == "off" or self.train_backend == "none" or not torch.is_grad_enabled():
            return False
        if x.requires_grad:
            return True
        return self.eval_autograd == "always" and any(p.requires_grad for p in self.parameters())

    @property
    def reduces_gradients(self) -> bool:
        """True when ``loss.backward()`` through this model already averages the gradients over the data-parallel ranks."""
        from .train_step import data_parallel_world
        return ((self.training or self.eval_autograd != "off") and self.train_backend == "native"
                and self.data_parallel != "off" and data_parallel_world() > 1)

    def _forward_train_native(self, x: torch.Tensor) -> torch.Tensor:
        """Training-kernel forward through libwunet_b200 (wunet_train_forward_ex / wunet_train_backward_ex behind a
        torch.autograd.Function): ``loss.backward()`` fills ``.grad`` of the parameters that require grad and of ``x`` when it
        requires grad; the caller's optimizer is used unchanged (trainer/trainer.py:34-38). Each block's BatchNorm follows
        its own container, as the reference's sub-modules do: in .train() it uses batch statistics and updates its running
        buffers with its own momentum (None: the cumulative factor 1 / num_batches_tracked) and counter; in .eval() it
        normalises by the running statistics and leaves them untouched. fp32 or, with ``train_precision="bf16"`` /
        ``"tf32"`` / ``"fp16_scaled"``, bf16 / tf32 / fp16 tensor-core convolutions (SURVEY §8f row N1, DESIGN §5.4).
        Forward hooks on the block containers receive the blocks' outputs as extra outputs of the autograd Function, so a loss
        on them back-propagates into the native backward."""
        plan = self._forward_hook_plan()
        if any(t.dtype in _HALF for t in self._param_tensors()):
            raise RuntimeError("libwunet_b200 needs contiguous float32 parameters on the input's device: the native training "
                               "step keeps float32 parameters. To train in 16 bits, train the float32 model with "
                               "Model(train_precision='bf16' or 'fp16_scaled') and call .half() / .to(torch.bfloat16) to deploy it.")
        self._check_input(x)
        B, _, T = x.shape
        blocks = self._blocks()
        bns = [blk[1] for blk in blocks]
        training = [bn.training for bn in bns]
        reducer = self._bn_sync_reducer() if any(training) else None
        if training[self.n_layers] and reducer is None and B * (T >> self.n_layers) == 1:
            # torch.nn.BatchNorm1d in training mode refuses batch statistics of one value per channel (here: the middle
            # block of a single frame of 2^n_layers samples); the reference raises this from self.middle
            raise ValueError("Expected more than 1 value per channel when training, got input size "
                             f"{torch.Size([B, self.n_layers * self.channels_interval, T >> self.n_layers])}")
        if not x.is_cuda:
            raise RuntimeError("wave_u_net_for_speech_enhancement_b200 has no CPU fallback: move the model and the "
                               "input to a CUDA (sm_90a) device")
        params = []
        for blk in blocks:
            params += [blk[0].weight, blk[0].bias, blk[1].weight, blk[1].bias]
        params += [self.out[0].weight, self.out[0].bias]
        for t in params:
            if t.device != x.device or t.dtype != torch.float32 or not t.is_contiguous():
                raise RuntimeError("libwunet_b200 needs contiguous float32 parameters on the input's device")
        # torch.nn.BatchNorm1d's exponential_average_factor of this step: momentum, or 1 / num_batches_tracked after the
        # increment when momentum is None (frozen blocks: unused)
        momenta = [0.0 if not tr else 1.0 / (int(bn.num_batches_tracked) + 1) if bn.momentum is None else float(bn.momentum)
                   for bn, tr in zip(bns, training)]
        train_momenta = {bn.momentum for bn, tr in zip(bns, training) if tr}
        trainable = [p.requires_grad for p in params]
        uniform = (all(training) or not any(training)) and len(train_momenta) <= 1 and None not in train_momenta and (
            all(trainable) or not any(trainable))
        flags = 0 if any(training) else _lib.TRAIN_FROZEN_BN
        if torch.backends.cudnn.deterministic or torch.are_deterministic_algorithms_enabled():
            flags |= _lib.TRAIN_DETERMINISTIC
        blocks_state = None if uniform else ([not tr for tr in training], momenta)
        if plan is None:
            y = _NativeTrainStep.apply(self, flags, reducer, blocks_state, self._aligned(x), *params)
        else:
            export = self._hook_levels(plan)
            y, *lv = _NativeTrainStepExport.apply(self, flags, reducer, blocks_state, tuple(export), self._aligned(x), *params)
        if not any(training):
            if plan is not None:
                self._fire_forward_hooks(plan, x, y, dict(zip(export, lv)))
            return y                                         # running statistics untouched: the folded copies stay valid
        for bn, tr in zip(bns, training):                    # torch.nn.BatchNorm1d bookkeeping
            if tr:
                bn.num_batches_tracked += 1
        # the kernels updated running_mean / running_var through raw pointers (no _version bump): drop the folded copies
        self._native.invalidate_weights()
        if plan is not None:
            self._fire_forward_hooks(plan, x, y, dict(zip(export, lv)))
        return y

    def _bn_sync_reducer(self):
        """The cross-rank sum of a batch-statistics native step, or None for per-rank statistics. It syncs exactly when
        ``nn.SyncBatchNorm`` would: every BatchNorm container is one (``nn.SyncBatchNorm.convert_sync_batchnorm(model)``),
        ``torch.distributed`` is initialised and their process group (WORLD when None) has more than one rank. Some
        containers converted and others not, or containers in different groups, raise ValueError. ``_bn_allreduce``, when
        set, is the reducer regardless (tests, tools/sync_bn_bench.py)."""
        if self._bn_allreduce is not None:
            return self._bn_allreduce
        bns = [blk[1] for blk in self._blocks()]
        synced = [isinstance(bn, nn.SyncBatchNorm) for bn in bns]
        if not any(synced):
            return None
        if not all(synced):
            raise ValueError(f"{sum(synced)} of the {len(bns)} BatchNorm containers are nn.SyncBatchNorm: the native training "
                             "step synchronises all of them or none (nn.SyncBatchNorm.convert_sync_batchnorm(model))")
        if len({id(bn.process_group) for bn in bns}) > 1:
            raise ValueError("the nn.SyncBatchNorm containers of this model use different process groups: the native "
                             "training step synchronises all of them over one group")
        group = bns[0].process_group
        if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) <= 1:
            return None
        return lambda buf: dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)

    def _check_input(self, x: torch.Tensor):
        """[B, 1, T], and float32 unless the parameters are all float16 (or all bfloat16): then of that dtype."""
        if x.dim() != 3 or x.size(1) != 1:
            raise RuntimeError(f"expected input of shape [B, 1, T], got {tuple(x.shape)}")
        pd = self._param_dtype()
        want = pd if pd in _HALF else torch.float32
        if x.dtype != want:
            raise RuntimeError(f"expected {str(want).replace('torch.', '')} input for a model whose parameters are "
                               f"{'of mixed dtypes' if pd is None else pd}, got {x.dtype}")

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
        plan = self._forward_hook_plan()
        self._check_input(x)
        empty = self._empty_batch(x)
        if empty is not None:
            if plan is not None:
                self._fire_forward_hooks(plan, x, empty, {i: self._level_empty(i, x) for i in self._hook_levels(plan)})
            return empty
        if not x.is_cuda:
            raise RuntimeError("wave_u_net_for_speech_enhancement_b200 has no CPU fallback: move the model and the "
                               "input to a CUDA (sm_90a) device")
        x_in, x = x, self._aligned(x)
        B, _, T = x.shape
        lib = _lib.load()
        with torch.cuda.device(x.device):
            ctx = self._context(x.device)
            self._sync_weights(ctx, x.device)
            prec = _lib.PRECISIONS[self.precision]
            ws = self._workspace(ctx, B, T, prec, x.device)
            y = torch.empty_like(x)
            stream = torch.cuda.current_stream(x.device).cuda_stream
            if plan is None:
                _lib.check(lib.wunet_forward_io(ctx, x.data_ptr(), y.data_ptr(), B, T, prec, _IO_DTYPES[x.dtype], ws.data_ptr(),
                                                ws.numel(), stream))
                return y
            nb = 2 * self.n_layers + 1
            levels = {i: self._level_empty(i, x) for i in self._hook_levels(plan)}
            mask = (ctypes.c_ubyte * nb)(*[1 if i in levels else 0 for i in range(nb)])
            outs = (ctypes.c_void_p * nb)(*[levels[i].data_ptr() if i in levels else None for i in range(nb)])
            _lib.check(lib.wunet_forward_export(ctx, x.data_ptr(), y.data_ptr(), B, T, prec, _IO_DTYPES[x.dtype], mask, outs,
                                                ws.data_ptr(), ws.numel(), stream))
        self._fire_forward_hooks(plan, x_in, y, levels)
        return y

    # ------------------------------------------------------------------------------------------
    # forward hooks on the block containers
    # ------------------------------------------------------------------------------------------
    def _hook_containers(self):
        """(name, module, block) of every container whose forward hooks the native forward fires, in the reference's call
        order (model/unet_basic.py:77-100: an encoder block's ``main`` returns inside the block's own call); block 2n+1 = out."""
        n = self.n_layers
        cs = []
        for i, e in enumerate(self.encoder):
            cs += [(f"encoder.{i}.main", e.main, i), (f"encoder.{i}", e, i)]
        cs.append(("middle", self.middle, n))
        for j, d in enumerate(self.decoder):
            cs += [(f"decoder.{j}.main", d.main, n + 1 + j), (f"decoder.{j}", d, n + 1 + j)]
        cs.append(("out", self.out, 2 * n + 1))
        return cs

    def _forward_hook_plan(self):
        """None when no forward hook fires on a block container: the forward then makes exactly the calls it makes without
        hooks. Otherwise the (name, module, block) whose hooks fire, in order. Raises for every hook on a sub-module that the
        native forward cannot honour, naming the module. A scan that finds nothing is remembered until the next hook handle is
        created anywhere (every registration creates one), so the hook-free forward pays one comparison."""
        if getattr(self, "_hook_free_at", None) == RemovableHandle.next_id:
            return None
        containers = self._hook_containers()
        ids = {id(m) for _, m, _ in containers}
        for name, m in self.named_modules():
            if m is self:
                continue
            what = f"{name} ({type(m).__name__})"
            if m._backward_hooks or m._backward_pre_hooks:
                raise NotImplementedError(f"{what} has a module backward hook: the native forward does not call the sub-modules, "
                                          "so their backward hooks are not supported. Register a tensor hook on the output a "
                                          "forward hook receives instead.")
            if m._forward_pre_hooks:
                raise NotImplementedError(f"{what} has a forward pre-hook: the native forward does not call the sub-modules, so "
                                          "forward pre-hooks on them are not supported (forward hooks on the block containers are)")
            if m._forward_hooks and id(m) not in ids:
                raise NotImplementedError(f"{what} has a forward hook: inside a block the native forward fuses convolution, "
                                          "BatchNorm and activation, so only forward hooks on encoder[i], encoder[i].main, middle, "
                                          "decoder[j], decoder[j].main and out are supported")
        fire = [c for c in containers if c[1]._forward_hooks or _nn_module._global_forward_hooks]
        if not fire:
            self._hook_free_at = RemovableHandle.next_id
            return None
        return fire

    def _hook_levels(self, plan):
        """The blocks whose outputs the hooks of ``plan`` receive, as their output or to build their input, ascending."""
        n = self.n_layers
        need = set()
        for _, _, b in plan:
            if b == 2 * n + 1:
                need.add(2 * n)                              # out's input: cat([decoder[n-1], x])
                continue
            need.add(b)
            if 0 < b <= n:
                need.add(b - 1)                              # previous output, decimated
            elif b > n:
                need.update((b - 1, 2 * n - b))              # previous output (upsampled) and the skip
        return sorted(need)

    def _level_empty(self, block: int, x: torch.Tensor) -> torch.Tensor:
        n, T = self.n_layers, x.shape[-1]
        L = T >> block if block <= n else T >> (2 * n - block)
        return torch.empty(x.shape[0], self._blocks()[block][0].out_channels, L, dtype=x.dtype, device=x.device)

    def _fire_forward_hooks(self, plan, x: torch.Tensor, y: torch.Tensor, levels) -> None:
        """Call the forward hooks of ``plan`` (global ones first, then the module's, as nn.Module.__call__ does) with
        ``(module, (input,), output)`` or, registered ``with_kwargs``, ``(module, (input,), {}, output)``. ``levels``: block ->
        output. A decoder block's input is built with torch (F.interpolate and torch.cat on the exported tensors), so its
        arithmetic is torch's. A hook that returns a value raises: the native forward cannot replace a block's output."""
        n = self.n_layers
        inputs = {}

        def block_input(b):
            if b not in inputs:
                if b == 0:
                    inputs[b] = x
                elif b <= n:
                    inputs[b] = levels[b - 1][:, :, ::2]
                elif b <= 2 * n:
                    up = F.interpolate(levels[b - 1], scale_factor=2, mode="linear", align_corners=True)
                    inputs[b] = torch.cat([up, levels[2 * n - b]], dim=1)
                else:
                    inputs[b] = torch.cat([levels[2 * n], x], dim=1)
            return inputs[b]

        g_hooks, g_kw = _nn_module._global_forward_hooks, _nn_module._global_forward_hooks_with_kwargs
        for name, m, b in plan:
            args, out = (block_input(b),), (y if b == 2 * n + 1 else levels[b])
            for hid, hook in (*g_hooks.items(), *m._forward_hooks.items()):
                if hid in m._forward_hooks_with_kwargs or hid in g_kw:
                    r = hook(m, args, {}, out)
                else:
                    r = hook(m, args, out)
                if r is not None:
                    raise RuntimeError(f"a forward hook on {name} ({type(m).__name__}) returned a value: the native forward "
                                       "cannot replace a block's output, so forward hooks must return None")

    @torch.no_grad()
    def forward_host(self, x_host: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """End-to-end form of enhancement.py:64-66 (``model(chunk).detach().cpu()``): host tensor in,
        host tensor out; H2D copy, kernels and D2H copy are enqueued by ``wunet_forward_host_io``.
        Parameters must already live on a CUDA device. Pinned tensors give full copy bandwidth. A 16-bit model takes and
        returns 16-bit tensors (half the copy bytes). Does not go through ``forward``: forward hooks do not fire."""
        self._check_input(x_host)
        if x_host.is_cuda:
            raise RuntimeError("forward_host takes a host tensor")
        if self.training or self._bn_any_training():
            raise NotImplementedError("forward_host is eval-only (model and every BatchNorm container in .eval())")
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
            _lib.check(_lib.load().wunet_forward_host_io(ctx, x_host.data_ptr(), out.data_ptr(), B, T,
                                                         _lib.PRECISIONS[self.precision], _IO_DTYPES[x_host.dtype]))
        return out

    @torch.no_grad()
    def forward_host_stream(self, batches, outs=None):
        """Streaming form of :meth:`forward_host` for many host batches (every chunk of every clip, enhancement.py:49-74):
        yields one output tensor per input batch, in order; H2D copy, kernels and D2H copy of consecutive batches overlap
        (two batches in flight). ``batches``: iterable of pinned ``[B,1,T]`` host tensors (float32, or the dtype of a 16-bit
        model) that must stay alive until their result has been yielded; ``outs``: optional iterable of pinned output
        tensors of the same dtype. Forward hooks do not fire."""
        if self.training or self._bn_any_training():
            raise NotImplementedError("forward_host_stream is eval-only (model and every BatchNorm container in .eval())")
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
                if out.dtype != x.dtype:
                    raise RuntimeError(f"output buffer is {out.dtype}, the input {x.dtype}")
                _lib.check(lib.wunet_stream_submit_io(ctx, x.data_ptr(), out.data_ptr(), B, T, prec, _IO_DTYPES[x.dtype],
                                                      ctypes.byref(ticket)))
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
