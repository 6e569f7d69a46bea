"""Fine-tuning with frozen layers in the native training step, host side (no GPU): which entry point the Python layer calls
for each per-block BatchNorm mode, momentum and requires_grad state, with which per-block arrays and gradient slots, the
BatchNorm bookkeeping, the gradient bucket with a trainable mask, and the C ABI surface. The library calls are recorded
through a fake binding."""
import contextlib
import ctypes
import os
import re
import types

import pytest
import torch
import torch.nn as nn

from wave_u_net_for_speech_enhancement_b200 import Model, _lib
from wave_u_net_for_speech_enhancement_b200.train_step import GradientBucket

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, CI = 4, 8
NB = 2 * N + 1


def header():
    return open(os.path.join(ROOT, "include", "wunet_b200.h")).read()


def slots(arr, n):
    """a ctypes pointer array (or None) -> one bool per entry: is the gradient slot set"""
    return [False] * n if arr is None else [bool(arr[i]) for i in range(n)]


class FakeLib:
    """Records the training calls: entry point, flags, per-block arrays and which gradient slots are set."""

    def __init__(self):
        self.calls = []

    def wunet_train_workspace_bytes_ex(self, c, B, T, prec, flags):
        return 64

    def wunet_train_forward_ex(self, *a):
        self.calls.append(("forward_ex", a[-1], a[13]))
        return 0

    def wunet_train_forward_blocks(self, *a):
        self.calls.append(("forward_blocks", a[-3], [int(v) for v in a[-2][:NB]], [round(float(v), 6) for v in a[-1][:NB]]))
        return 0

    def _backward(self, name, a, extra):
        g = {k: slots(a[10 + j], NB) for j, k in enumerate(("w", "b", "gamma", "beta"))}
        g["out"] = [bool(a[14]), bool(a[15])]
        self.calls.append((name, a[20], a[22], bool(a[19]), g) + extra)
        return 0

    def wunet_train_backward_ex(self, *a):
        return self._backward("backward_ex", a, ())

    def wunet_train_backward_blocks(self, *a):
        return self._backward("backward_blocks", a[:-1], ([int(v) for v in a[-1][:NB]],))

    def wunet_last_error(self):
        return b"fake failure"


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda d=None: types.SimpleNamespace(cuda_stream=0))
    monkeypatch.setattr(Model, "_context", lambda self, d: None)
    return lib


def bns(m):
    return [blk[1] for blk in m._blocks()]


def step(m, x=None):
    x = torch.zeros(2, 1, 256) if x is None else x
    y = m(x)
    if y.grad_fn is not None:
        y.sum().backward()
    return y


def test_uniform_states_keep_the_ex_calls(fake):
    m = Model(N, CI).train()
    step(m)
    assert fake.calls[0] == ("forward_ex", 0, pytest.approx(0.1))
    assert fake.calls[1][:4] == ("backward_ex", -1, 0, False) and all(all(v) for v in fake.calls[1][4].values())
    assert all(int(bn.num_batches_tracked) == 1 for bn in bns(m))
    # a model in .train() whose containers are all in .eval(): the frozen step, no bookkeeping
    fake.calls.clear()
    for bn in bns(m):
        bn.eval()
    step(m)
    assert [c[:2] for c in fake.calls] == [("forward_ex", _lib.TRAIN_FROZEN_BN), ("backward_ex", -1)]
    assert fake.calls[1][2] == _lib.TRAIN_FROZEN_BN
    assert all(int(bn.num_batches_tracked) == 1 for bn in bns(m))
    # an .eval() model recording a graph for x.grad: the frozen step, x and every parameter
    fake.calls.clear()
    m.eval()
    step(m, torch.zeros(2, 1, 256, requires_grad=True))
    assert [c[:2] for c in fake.calls] == [("forward_ex", _lib.TRAIN_FROZEN_BN), ("backward_ex", -1)]
    assert fake.calls[1][2] == _lib.TRAIN_FROZEN_BN and fake.calls[1][3]
    # ... and with every parameter frozen: the input gradient only
    fake.calls.clear()
    m.requires_grad_(False)
    step(m, torch.zeros(2, 1, 256, requires_grad=True))
    assert [c[:3] for c in fake.calls] == [("forward_ex", _lib.TRAIN_FROZEN_BN, pytest.approx(0.1)),
                                           ("backward_ex", -1, _lib.TRAIN_FROZEN_BN | _lib.TRAIN_NO_PARAM_GRADS)]


def test_mixed_batchnorm_modes(fake):
    m = Model(N, CI).train()
    for e in m.encoder:
        e.main[1].eval()
    step(m)
    frozen = [1] * N + [0] * (N + 1)
    assert fake.calls[0] == ("forward_blocks", 0, frozen, [0.0] * N + [0.1] * (N + 1))
    name, part, flags, dx, g, bf = fake.calls[1]
    assert (name, part, flags, dx, bf) == ("backward_blocks", -1, 0, False, frozen)
    assert all(all(v) for v in g.values())
    assert [int(bn.num_batches_tracked) for bn in bns(m)] == [0] * N + [1] * (N + 1)


def test_per_block_momenta_and_none_over_several_steps(fake):
    m = Model(N, CI).train()
    for i, bn in enumerate(bns(m)):
        bn.momentum = None if i % 3 == 0 else 0.05 * (i + 1)
    for k in range(1, 4):
        step(m)
        call = fake.calls[2 * (k - 1)]
        assert call[0] == "forward_blocks" and call[2] == [0] * NB
        want = [round(1.0 / k if i % 3 == 0 else 0.05 * (i + 1), 6) for i in range(NB)]
        assert call[3] == pytest.approx(want)
    assert all(int(bn.num_batches_tracked) == 3 for bn in bns(m))


def test_partial_requires_grad(fake):
    m = Model(N, CI).train()
    m.encoder.requires_grad_(False)
    m.middle.requires_grad_(False)
    step(m)
    assert fake.calls[0] == ("forward_blocks", 0, [0] * NB, [0.1] * NB)
    name, part, flags, dx, g, bf = fake.calls[1]
    assert (name, part, flags, dx, bf) == ("backward_blocks", -1, 0, False, [0] * NB)
    for k in ("w", "b", "gamma", "beta"):
        assert g[k] == [False] * (N + 1) + [True] * N, k
    assert g["out"] == [True, True]
    for k, p in m.named_parameters():
        assert (p.grad is None) == k.startswith(("encoder.", "middle.")), k
    # head only, one head parameter frozen
    fake.calls.clear()
    m.zero_grad(set_to_none=True)
    m.decoder.requires_grad_(False)
    m.out[0].bias.requires_grad_(False)
    step(m)
    g = fake.calls[1][4]
    assert not any(any(g[k]) for k in ("w", "b", "gamma", "beta")) and g["out"] == [True, False]
    assert m.out[0].weight.grad is not None and m.out[0].bias.grad is None


def test_eval_model_with_one_container_in_train_mode(fake):
    m = Model(N, CI).eval()
    m.middle[1].train()
    y = m(torch.zeros(2, 1, 256))
    assert y.grad_fn is None and not y.requires_grad                    # eval_autograd="input", x needs no grad: detached
    frozen = [1] * NB
    frozen[N] = 0
    assert fake.calls == [("forward_blocks", 0, frozen, [0.0] * N + [0.1] + [0.0] * N)]
    assert [int(bn.num_batches_tracked) for bn in bns(m)] == [0] * N + [1] + [0] * N
    # with a graph (x requires grad): the backward of the same per-block step
    fake.calls.clear()
    step(m, torch.zeros(2, 1, 256, requires_grad=True))
    assert fake.calls[1][:4] == ("backward_blocks", -1, 0, True) and fake.calls[1][5] == frozen


def test_host_forwards_refuse_a_container_in_train_mode():
    m = Model(N, CI).eval()
    m.middle[1].train()
    with pytest.raises(NotImplementedError, match="eval-only"):
        m.forward_host(torch.zeros(2, 1, 256))
    with pytest.raises(NotImplementedError, match="eval-only"):
        next(m.forward_host_stream([torch.zeros(2, 1, 256)]))


def test_one_value_per_channel_checks_only_a_middle_block_in_train_mode(fake):
    x = torch.zeros(1, 1, 16)                                            # L = 1 at the middle block
    m = Model(N, CI).train()
    m.middle[1].eval()
    step(m, x)
    assert fake.calls[0][0] == "forward_blocks"
    m.middle[1].train()
    m.encoder[0].main[1].eval()
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        m(x)


def test_split_backward_passes_the_mask_and_dx_to_both_parts(fake, monkeypatch):
    import wave_u_net_for_speech_enhancement_b200.train_step as ts
    monkeypatch.setattr(ts, "data_parallel_world", lambda: 2)
    monkeypatch.setattr(GradientBucket, "reduce_part", lambda self, k, group=None: None)
    monkeypatch.setattr(GradientBucket, "finish", lambda self: None)
    m = Model(N, CI).train()
    m.encoder.requires_grad_(False)
    step(m, torch.zeros(2, 1, 256, requires_grad=True))
    assert [(c[0], c[1], c[3]) for c in fake.calls[1:]] == [("backward_blocks", 0, True), ("backward_blocks", 1, True)]


def shapes(m):
    return [p.shape for p in m.parameters()]


def test_bucket_without_mask_keeps_the_layout():
    m = Model(N, CI)
    b = GradientBucket(shapes(m), NB, "cpu")
    # backward-completion order: head, decoders last to first (part 0), middle, encoders last to first (part 1)
    order = [4 * NB, 4 * NB + 1] + [4 * i + k for i in range(NB - 1, N, -1) for k in range(4)]
    n0 = len(order)
    order += [4 * i + k for i in range(N, -1, -1) for k in range(4)]
    off, want = 0, {}
    for j, i in enumerate(order):
        if j == n0:
            off = (off + 127) // 128 * 128
            assert b.split == off
        want[i] = off
        off += (shapes(m)[i].numel() + 3) // 4 * 4
    assert b.flat.numel() == off
    assert {i: v.storage_offset() for i, v in enumerate(b.views)} == want


def test_bucket_with_mask_holds_only_trainable_parameters():
    m = Model(N, CI)
    sh = shapes(m)
    mask = [i >= 4 * (N + 1) for i in range(len(sh))]                  # decoders + head: part 1 empty
    b = GradientBucket(sh, NB, "cpu", trainable=mask)
    assert all((v is None) != t for v, t in zip(b.views, mask))
    assert b.part(1).numel() == 0
    assert b.flat.numel() == sum((sh[i].numel() + 3) // 4 * 4 for i in range(len(sh)) if mask[i])
    full = GradientBucket(sh, NB, "cpu")
    assert [full.views[i].storage_offset() for i in range(len(sh)) if mask[i]] == \
        [b.views[i].storage_offset() for i in range(len(sh)) if mask[i]]        # the same prefix of the layout
    enc = [i < 4 * N for i in range(len(sh))]                             # encoders only: part 0 empty
    b2 = GradientBucket(sh, NB, "cpu", trainable=enc)
    assert b2.split == 0 and b2.part(0).numel() == 0 and b2.part(1).numel() == b2.flat.numel() > 0
    with pytest.raises(ValueError):
        GradientBucket(sh, NB, "cpu", trainable=mask[:-1])


def test_header_exports_and_flag_set():
    h = header()
    for fn in ("wunet_train_forward_blocks", "wunet_train_backward_blocks"):
        assert re.search(rf"int {fn}\(wunet_ctx \*ctx,", h), fn
        assert fn in _lib.EXPORTED_SYMBOLS
    assert re.search(r"const unsigned char \*bn_frozen,\s*const float \*momenta\);", h)
    assert re.search(r"int precision, int flags, const unsigned char \*bn_frozen\);", h)
    flags = dict(re.findall(r"#define\s+(WUNET_TRAIN_[A-Z_]+)\s+(\d+)", h))
    assert flags == {"WUNET_TRAIN_FROZEN_BN": "1", "WUNET_TRAIN_NO_PARAM_GRADS": "2", "WUNET_TRAIN_DETERMINISTIC": "16"}


def test_sync_reducer_is_not_consulted_when_every_container_is_frozen(fake):
    m = nn.SyncBatchNorm.convert_sync_batchnorm(Model(N, CI)).train()
    m._bn_allreduce = lambda buf: pytest.fail("frozen BatchNorm must not synchronise")
    for bn in bns(m):
        bn.eval()
    step(m)
    assert fake.calls[0][:2] == ("forward_ex", _lib.TRAIN_FROZEN_BN)
