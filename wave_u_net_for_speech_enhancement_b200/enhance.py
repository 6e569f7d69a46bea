"""
Chunk batching for inference (SURVEY §8f row N2): the reference's ``enhancement.py:49-74`` (and the validation loop,
``trainer/trainer.py:58-79``) zero-pads every clip to a multiple of ``sample_length``, splits it into 16384-sample chunks
and pushes them through the model ONE chunk at a time with a device→host sync each. Chunks are independent in eval mode,
so this module stacks the chunks of many clips on the batch axis and streams the batches through
``Model.forward_host_stream`` (H2D copy / kernels / D2H copy of consecutive batches overlap), then re-assembles and trims
every clip exactly like the reference loop does (``enhancement.py:68-71``).
"""
from __future__ import annotations

import ctypes
import os
from typing import Callable, Iterable, List, Sequence, Tuple

import numpy as np
import torch

from . import _lib


class _PinnedPool:
    """Grow-only pinned staging buffers, reused across calls: allocating page-locked memory costs milliseconds, a forward of
    a few hundred frames costs one. Single-threaded use (every result is copied out of the pool before the call returns)."""

    def __init__(self):
        self._buf = {}

    def get(self, name: str, frames: int, sample_length: int, pin: bool, dtype: torch.dtype = torch.float32) -> torch.Tensor:
        key = (name, sample_length, pin, dtype)
        t = self._buf.get(key)
        if t is None or t.shape[0] < frames:
            t = torch.empty(max(frames, 1), 1, sample_length, dtype=dtype)
            if pin:
                t = t.pin_memory()
            self._buf[key] = t
        return t[:frames]


_POOL = _PinnedPool()


HOST_THREADS = max(1, min(8, (os.cpu_count() or 1) // 2))   # host threads of the native framing / trimming passes


def _clip_table(waveforms: Sequence[np.ndarray], sample_length: int):
    """Contiguous clips (float32, or int16 PCM kept as it is), their lengths, and per clip (first_frame, n_frames, length)."""
    clips, index, total = [], [], 0
    for w in waveforms:
        a = np.asarray(w)
        if a.ndim != 1:
            raise ValueError("waveforms must be 1-D")
        if a.dtype != np.int16:
            a = np.ascontiguousarray(a, dtype=np.float32)
        else:
            a = np.ascontiguousarray(a)
        n = int(a.shape[0])
        nf = max(1, -(-n // sample_length))
        clips.append(a)
        index.append((total, nf, n))
        total += nf
    return clips, index, total


def _ptr_array(arrays):
    return (ctypes.c_void_p * len(arrays))(*[a.ctypes.data for a in arrays])


_IO = {torch.float32: _lib.IO_F32, torch.float16: _lib.IO_F16, torch.bfloat16: _lib.IO_BF16}


def frame_clips(waveforms: Sequence[np.ndarray], sample_length: int = 16384, pin: bool = True, round_to: int = 1,
                dtype: torch.dtype = torch.float32) -> Tuple[torch.Tensor, List[Tuple[int, int, int]]]:
    """Zero-pad each 1-D waveform to a multiple of ``sample_length`` (enhancement.py:57-59) and split it into chunks
    (enhancement.py:62). Returns the stacked chunks ``[N,1,sample_length]`` (float32; a view of a pooled pinned staging
    buffer if requested, valid until the next call) and, per clip, ``(first_frame, n_frames, original_length)``.
    ``N`` is the number of chunks rounded up to a multiple of ``round_to`` (silent frames, so that every batch of the stream
    has the same size). float32 clips are copied, int16 PCM clips (a wav file's samples) are converted like the reference's
    loader does (sample / 32768); both by the library's multi-threaded ``wunet_frame_clips_*`` (row N4). ``dtype`` float16
    or bfloat16 (a half model's input): each sample is computed in fp32 as above and rounded once to it."""
    clips, index, total = _clip_table(waveforms, sample_length)
    kinds = {c.dtype for c in clips}
    if len(kinds) > 1:
        raise ValueError("mixing int16 and float32 clips in one call is not supported")
    padded = -(-max(total, 1) // round_to) * round_to
    if dtype not in _IO:
        raise ValueError(f"frames of dtype {dtype} are not supported (float32, float16, bfloat16)")
    frames = _POOL.get("in", padded, sample_length, pin and torch.cuda.is_available(), dtype)
    lib = _lib.load()
    lens = (ctypes.c_longlong * len(clips))(*[c.shape[0] for c in clips])
    i16 = kinds == {np.dtype(np.int16)}
    args = (_ptr_array(clips), lens, len(clips), sample_length, frames.data_ptr(), padded, HOST_THREADS)
    if dtype == torch.float32:
        _lib.check((lib.wunet_frame_clips_i16 if i16 else lib.wunet_frame_clips_f32)(*args))
    else:
        _lib.check((lib.wunet_frame_clips_i16_io if i16 else lib.wunet_frame_clips_f32_io)(*args, _IO[dtype]))
    return frames, index


def unframe_clips(frames: torch.Tensor, index: List[Tuple[int, int, int]], copy: bool = True) -> List[np.ndarray]:
    """Concatenate each clip's chunks and drop the padding (enhancement.py:68-71). A clip's chunks are consecutive rows, so
    with ``copy=False`` the results are views of ``frames`` (valid as long as that buffer is not reused)."""
    sample_length = int(frames.shape[-1])
    if not copy:
        flat = frames.view(-1).numpy()
        return [flat[f0 * sample_length:f0 * sample_length + n] for (f0, _nf, n) in index]
    out = [np.empty(n, dtype=np.float32) for (_f0, _nf, n) in index]
    lens = (ctypes.c_longlong * len(out))(*[n for (_f0, _nf, n) in index])
    _lib.check(_lib.load().wunet_unframe_clips_f32(frames.data_ptr(), _ptr_array(out), lens, len(out), sample_length,
                                                   int(frames.shape[0]), HOST_THREADS))
    return out


def enhance_waveforms(model, waveforms: Sequence[np.ndarray], sample_length: int = 16384, batch_frames: int = 256,
                      stream_fn: Callable[[Iterable[torch.Tensor], Iterable[torch.Tensor]], Iterable[torch.Tensor]] = None,
                      copy: bool = True) -> List[np.ndarray]:
    """Enhance a list of 1-D waveforms (float32, or int16 PCM); returns the enhanced float32 waveforms (same lengths).
    ``copy=False`` returns views of the pooled pinned output buffer instead of fresh arrays: valid until the next call, for a
    caller that consumes every clip at once the way enhancement.py:73-74 writes it to disk.

    ``model`` is a ``wave_u_net_for_speech_enhancement_b200.Model`` on a CUDA device in eval mode. ``stream_fn`` (tests
    only) replaces ``model.forward_host_stream``. A half model (``model.half()`` / ``.to(torch.bfloat16)``) gets frames of
    its dtype (half the copy bytes); its 16-bit output is widened to the float32 waveforms returned. It streams through
    ``Model.forward_host_stream``, not ``forward``: forward hooks on the model's blocks do not fire."""
    _clips, _index, total = _clip_table(waveforms, sample_length)
    B = max(1, min(batch_frames, total))
    dtype = model._param_dtype() if hasattr(model, "_param_dtype") else None      # stream_fn tests may pass no model
    dtype = dtype if dtype in (torch.float16, torch.bfloat16) else torch.float32
    # the batch size stays constant (one plan / workspace): the last batch is filled up with silent frames by the framing pass
    frames, index = frame_clips(waveforms, sample_length, round_to=B, dtype=dtype)
    padded = frames.shape[0]
    out = _POOL.get("out", padded, sample_length, frames.is_pinned(), dtype)
    batches = [frames[i:i + B] for i in range(0, padded, B)]
    outs = [out[i:i + B] for i in range(0, padded, B)]
    fn = stream_fn if stream_fn is not None else model.forward_host_stream
    for _ in fn(batches, outs):
        pass
    if dtype != torch.float32:
        wide = _POOL.get("out_f32", padded, sample_length, False)
        wide.copy_(out)                                    # exact
        out = wide
    return unframe_clips(out, index, copy)


# ---------------------------------------------------------------------------------------------------------------------------
# several GPUs (BASELINE.json configs[3]: batch 1024 sharded over 8 GPUs): one process per GPU, clips dealt to the ranks,
# no collective on the data path (frames are independent in eval mode; SURVEY §8e)
# ---------------------------------------------------------------------------------------------------------------------------
def shard_clips(lengths: Sequence[int], world: int, sample_length: int = 16384) -> List[List[int]]:
    """Deal clips to ``world`` ranks so that every rank gets about the same number of 16384-sample frames: longest clip
    first onto the least loaded rank (ties: lowest rank); every rank's list is returned in ascending clip order.
    Deterministic, so every rank computes the same assignment without communicating."""
    frames = [max(1, -(-int(n) // sample_length)) for n in lengths]
    load = [0] * world
    out: List[List[int]] = [[] for _ in range(world)]
    for i in sorted(range(len(frames)), key=lambda i: (-frames[i], i)):
        r = min(range(world), key=lambda r: (load[r], r))
        out[r].append(i)
        load[r] += frames[i]
    return [sorted(ix) for ix in out]


def enhance_waveforms_sharded(model, waveforms: Sequence[np.ndarray], rank: int, world: int, sample_length: int = 16384,
                              batch_frames: int = 256, stream_fn=None, gather: bool = False, copy: bool = True):
    """This rank's share of :func:`enhance_waveforms` over ``world`` ranks (``enhancement.py:49-74`` sharded by clip).

    Returns ``{clip index: enhanced waveform}`` for the clips of this rank; with ``gather=True`` (needs an initialised
    ``torch.distributed`` group) rank 0 gets the full list in clip order — the only communication, and only of results
    (what a single writer of the output directory, ``enhancement.py:73-74``, needs) — and the other ranks get None."""
    mine = shard_clips([int(np.asarray(w).shape[-1]) for w in waveforms], world, sample_length)[rank]
    local = enhance_waveforms(model, [waveforms[i] for i in mine], sample_length, batch_frames, stream_fn,
                              copy or gather) if mine else []
    result = dict(zip(mine, local))
    if not gather:
        return result
    import torch.distributed as dist
    parts = [None] * world if rank == 0 else None
    dist.gather_object(result, parts, dst=0)
    if rank != 0:
        return None
    merged = {}
    for p in parts:
        merged.update(p)
    return [merged[i] for i in range(len(waveforms))]
