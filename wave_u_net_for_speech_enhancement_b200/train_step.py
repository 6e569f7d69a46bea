"""Data-parallel training step around the drop-in model (SURVEY.md §8f row N1 / config 5).

The reference wraps the model in single-process ``nn.DataParallel`` (trainer/base_trainer.py:26-27): every step it scatters
the batch, replicates the parameters, runs per-replica forwards (BatchNorm statistics per replica) and sums the replica
gradients on GPU 0. Here it is one process per GPU: each rank steps its own shard of the batch and the gradients are
averaged over ONE flat bucket (NCCL on GPUs, gloo in the CPU tests) before the caller's unchanged optimizer step — the mean
over ranks of per-shard mean losses is the reference's mean loss over the whole batch when the shards are equal. BatchNorm
statistics stay per rank, as they stay per replica in the reference (only replica 0's survive there; rank 0 writes the
checkpoint here), unless the model is converted with ``nn.SyncBatchNorm.convert_sync_batchnorm``: the native step then
computes them over every rank's frames (three small all-reduces per block, on the current stream), and with equal shards the
averaged step equals the single-process step on the concatenated batch.

The bucket is laid out in the order the backward pass FINISHES the gradients (head, decoder blocks last to first, middle,
encoder blocks last to first) and cut in two parts at the decoder / middle boundary: the native backward
(``wunet_train_backward_part``) hands part 0 to the collective while part 1 is still being computed, so the all-reduce of the
first half overlaps the second half of the backward; logically it is one all-reduce of one 40.5 MB bucket.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence

import torch
import torch.distributed as dist


def data_parallel_world() -> int:
    """Ranks that share the gradient all-reduce: the default process group's size, 1 when torch.distributed is not set up."""
    if not dist.is_available() or not dist.is_initialized():
        return 1
    return dist.get_world_size()


class GradientBucket:
    """Flat fp32 gradient buffer of one model, in backward-completion order.

    ``shapes``: parameter shapes in the model's ``parameters()`` order (4 per conv block — conv.weight, conv.bias, bn.weight,
    bn.bias — for the ``nblocks`` blocks in forward order, then out.weight, out.bias; model/unet_basic.py:33-75).
    ``views[i]`` is the slice of the flat buffer that holds parameter i's gradient.

    ``trainable`` (optional, one bool per parameter): only these get a slot, in the same order; the others' views are None, and
    a part with no trainable parameter is not all-reduced. Without it every parameter has one (the layout does not change)."""

    def __init__(self, shapes: Sequence[torch.Size], nblocks: int, device, dtype=torch.float32,
                 trainable: Optional[Sequence[bool]] = None):
        if len(shapes) != 4 * nblocks + 2:
            raise ValueError(f"expected {4 * nblocks + 2} parameter shapes, got {len(shapes)}")
        if trainable is not None and len(trainable) != len(shapes):
            raise ValueError(f"expected {len(shapes)} trainable flags, got {len(trainable)}")
        keep = (lambda i: True) if trainable is None else (lambda i: bool(trainable[i]))     # noqa: E731
        n_enc_mid = (nblocks + 1) // 2                        # encoder blocks + middle = n + 1 of the 2n + 1 blocks
        order: List[int] = [i for i in (4 * nblocks, 4 * nblocks + 1) if keep(i)]      # head first ...
        for blk in range(nblocks - 1, n_enc_mid - 1, -1):     # ... decoder blocks, last to first: part 0
            order += [4 * blk + k for k in range(4) if keep(4 * blk + k)]
        n_part0 = len(order)
        for blk in range(n_enc_mid - 1, -1, -1):              # middle, encoder blocks last to first: part 1
            order += [4 * blk + k for k in range(4) if keep(4 * blk + k)]
        sizes = [int(torch.Size(shapes[i]).numel()) for i in order]
        pad = lambda n, a: (n + a - 1) // a * a             # noqa: E731 - every gradient starts 16-byte aligned
        offs, off = [], 0
        for j, n in enumerate(sizes):
            if j == n_part0:
                off = pad(off, 128)                           # part 1 starts on a 512-byte boundary
                self.split = off
            offs.append(off)
            off += pad(n, 4)
        if n_part0 == len(order):                            # no trainable parameter in part 1
            self.split = off
        self.flat = torch.zeros(off, dtype=dtype, device=device)      # zeros: the padding takes part in the all-reduce
        self.views: List[Optional[torch.Tensor]] = [None] * len(shapes)
        for i, n, o in zip(order, sizes, offs):
            self.views[i] = self.flat[o:o + n].view(shapes[i])
        self._works = []
        self._needs_div = False

    def part(self, k: int) -> torch.Tensor:
        return self.flat[:self.split] if k == 0 else self.flat[self.split:]

    def reduce_part(self, k: int, group=None) -> None:
        """Start averaging part k over the ranks (asynchronous: the collective is ordered after the work already enqueued
        on the current stream and overlaps what is enqueued next)."""
        if data_parallel_world() == 1 or self.part(k).numel() == 0:
            return
        backend = dist.get_backend(group)
        if backend == "nccl":
            self._works.append(dist.all_reduce(self.part(k), op=dist.ReduceOp.AVG, group=group, async_op=True))
        else:                                                # gloo (CPU tests): no AVG
            self._works.append(dist.all_reduce(self.part(k), op=dist.ReduceOp.SUM, group=group, async_op=True))
            self._needs_div = True

    def finish(self) -> None:
        """Order everything enqueued after this call behind the collectives (stream-level wait on CUDA, no host sync)."""
        for w in self._works:
            w.wait()
        self._works = []
        if self._needs_div:
            self.flat.div_(data_parallel_world())
            self._needs_div = False


def allreduce_gradients(params: Iterable[torch.nn.Parameter], nblocks: Optional[int] = None) -> None:
    """Average ``.grad`` of the given parameters over all ranks, in place, through one flat bucket. For models whose backward
    does not reduce by itself (``Model(train_backend="torch")``, the reference module): gradients are copied into the bucket,
    reduced and copied back."""
    if data_parallel_world() == 1:
        return
    ps = [p for p in params]
    if any(p.grad is None for p in ps):
        raise RuntimeError("allreduce_gradients: every parameter needs a gradient (call it after loss.backward())")
    nb = nblocks if nblocks is not None else (len(ps) - 2) // 4
    bucket = GradientBucket([p.shape for p in ps], nb, ps[0].grad.device, ps[0].grad.dtype)
    for p, v in zip(ps, bucket.views):
        v.copy_(p.grad)
    bucket.reduce_part(0)
    bucket.reduce_part(1)
    bucket.finish()
    for p, v in zip(ps, bucket.views):
        p.grad.copy_(v)


def train_step(model: torch.nn.Module, optimizer: torch.optim.Optimizer, loss_function, mixture: torch.Tensor,
               clean: torch.Tensor) -> float:
    """trainer/trainer.py:34-38 for one rank's shard, plus the gradient all-reduce; returns this rank's loss. The native
    training backend reduces inside ``loss.backward()`` (overlapped with the backward kernels); other backends are reduced
    here after the backward."""
    optimizer.zero_grad()
    enhanced = model(mixture)
    loss = loss_function(clean, enhanced)
    loss.backward()
    if not getattr(model, "reduces_gradients", False):
        allreduce_gradients(model.parameters())
    optimizer.step()
    return float(loss.detach())
