"""Synchronised BatchNorm (nn.SyncBatchNorm) in the native training step, host side (no GPU): the C ABI surface, the state_dict
of a converted model, and when the Python layer installs the BatchNorm all-reduce hook. The library calls are recorded
through a fake binding; torch.distributed is replaced by stubs where a world of two ranks is needed."""
import contextlib
import inspect
import json
import os
import re
import types

import pytest
import torch
import torch.distributed as dist
import torch.nn as nn

from wave_u_net_for_speech_enhancement_b200 import Model, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header():
    return open(os.path.join(ROOT, "include", "wunet_b200.h")).read()


def test_entry_point_and_typedef_are_declared_and_exported():
    h = header()
    assert re.search(r"typedef int \(\*wunet_bn_allreduce_fn\)\(void \*user,\s*double \*buf,\s*size_t count,\s*void \*stream\);", h)
    assert re.search(r"int wunet_train_set_bn_allreduce\(wunet_ctx \*ctx,\s*wunet_bn_allreduce_fn fn,\s*void \*user,\s*double \*buf,"
                     r"\s*size_t capacity\);", h)
    assert "wunet_train_set_bn_allreduce" in _lib.EXPORTED_SYMBOLS


def test_flag_set_and_constructor_are_unchanged():
    flags = dict(re.findall(r"#define\s+(WUNET_TRAIN_[A-Z_]+)\s+(\d+)", header()))
    assert flags == {"WUNET_TRAIN_FROZEN_BN": "1", "WUNET_TRAIN_NO_PARAM_GRADS": "2", "WUNET_TRAIN_DETERMINISTIC": "16"}
    params = inspect.signature(Model.__init__).parameters
    assert [(p.name, p.default) for p in list(params.values())[1:]] == [
        ("n_layers", 12), ("channels_interval", 24), ("precision", "fp32_tc"), ("train_backend", "native"),
        ("data_parallel", "auto"), ("train_precision", "fp32"), ("eval_autograd", "input")]


def test_converted_model_keeps_state_dict_and_parameter_order():
    surface = json.load(open(os.path.join(ROOT, "tests", "golden", "state_dict_surface.json")))
    m = Model()
    order = [k for k, _ in m.named_parameters()]
    s = nn.SyncBatchNorm.convert_sync_batchnorm(m)
    assert s is m and sum(isinstance(b, nn.SyncBatchNorm) for b in s.modules()) == 25
    sd = s.state_dict()
    assert [[k, list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd.items()] == surface["state_dict"]
    assert [k for k, _ in s.named_parameters()] == order
    assert all(b[1] is not None and isinstance(b[1], nn.SyncBatchNorm) for b in s._blocks())


class FakeLib:
    """Records the training calls and the hook installs; the forward calls an installed hook once per pass like the library
    (block 0 only: C = its Cout), so the reducer plumbing runs end to end."""

    def __init__(self, cout0):
        self.calls, self.hook, self.cout0 = [], None, cout0

    def wunet_train_workspace_bytes_ex(self, c, B, T, prec, flags):
        return 64

    def wunet_train_set_bn_allreduce(self, c, fn, user, buf, capacity):
        self.calls.append(("set", bool(fn), capacity))
        self.hook = (fn, buf) if fn else None
        return 0

    def wunet_train_forward_ex(self, c, x, y, B, T, *rest):
        self.calls.append(("forward_ex", B, rest[-1]))
        if self.hook is not None:
            fn, buf = self.hook
            C = self.cout0
            for ptr, count in ((buf, C + 1), (buf + 8 * (C + 1), C)):
                rc = fn(None, ptr, count, None)
                self.calls.append(("hook", count, rc))
                if rc:
                    return -2                    # WUNET_ECUDA
        return 0

    def wunet_last_error(self):
        return b"fake failure"


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib(8)
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda d=None: types.SimpleNamespace(cuda_stream=0))
    monkeypatch.setattr(Model, "_context", lambda self, d: None)
    return lib


@pytest.fixture
def world(monkeypatch):
    """torch.distributed stubs: sizes per group object (None = WORLD), every all_reduce recorded (buffer length, op, group)."""
    state = types.SimpleNamespace(sizes={None: 2}, reduced=[], initialised=True)
    monkeypatch.setattr(dist, "is_available", lambda: True)
    monkeypatch.setattr(dist, "is_initialized", lambda: state.initialised)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: state.sizes[group])

    def all_reduce(t, op=None, group=None, async_op=False):
        state.reduced.append((t.numel(), t.dtype, op, group))
        t.mul_(2)                                        # two ranks holding the same sums
    monkeypatch.setattr(dist, "all_reduce", all_reduce)
    return state


def converted(**kw):
    return nn.SyncBatchNorm.convert_sync_batchnorm(Model(4, 8, **kw))


def test_world_of_two_installs_the_hook_around_the_forward(fake, world):
    m = converted().train()
    y = m(torch.zeros(2, 1, 256))
    assert y.grad_fn is not None
    need = 2 * 4 * 8 + 1
    assert fake.calls == [("set", True, need), ("forward_ex", 2, 0), ("hook", 9, 0), ("hook", 8, 0), ("set", False, 0)]
    assert world.reduced == [(9, torch.float64, dist.ReduceOp.SUM, None), (8, torch.float64, dist.ReduceOp.SUM, None)]


def test_explicit_group_is_used(fake, world):
    g = object()
    world.sizes[g] = 3
    m = Model(4, 8)
    m = nn.SyncBatchNorm.convert_sync_batchnorm(m, process_group=g).train()
    m(torch.zeros(2, 1, 256))
    assert [r[3] for r in world.reduced] == [g, g]


@pytest.mark.parametrize("case", ["world1", "no_dist", "eval", "not_converted"])
def test_no_hook(fake, world, case):
    m = Model(4, 8) if case == "not_converted" else converted()
    if case == "world1":
        world.sizes[None] = 1
    if case == "no_dist":
        world.initialised = False
    x = torch.zeros(2, 1, 256, requires_grad=case == "eval")
    m.train(case != "eval")
    y = m(x)
    assert y.grad_fn is not None
    want = _lib.TRAIN_FROZEN_BN if case == "eval" else 0
    assert fake.calls == [("forward_ex", 2, want)] and world.reduced == []


def test_frozen_bn_never_syncs_even_with_the_seam(fake, world):
    m = converted().eval()
    m._bn_allreduce = lambda buf: pytest.fail("frozen BatchNorm must not synchronise")
    m(torch.zeros(2, 1, 256, requires_grad=True))
    assert fake.calls == [("forward_ex", 2, _lib.TRAIN_FROZEN_BN)]


def test_seam_forces_the_sync_path_without_dist(fake, world):
    world.initialised = False
    seen = []
    m = Model(4, 8).train()
    m._bn_allreduce = lambda buf: seen.append((buf.numel(), buf.dtype))
    m(torch.zeros(2, 1, 256))
    assert seen == [(9, torch.float64), (8, torch.float64)] and world.reduced == []


def test_one_value_per_channel_is_legal_only_when_synced(fake, world):
    x = torch.zeros(1, 1, 16)                            # n = 4: L = 1 at the middle block
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        Model(4, 8).train()(x)
    converted().train()(x)
    assert ("forward_ex", 1, 0) in fake.calls


def test_partial_conversion_raises(fake, world):
    m = Model(4, 8)
    m.middle[1] = nn.SyncBatchNorm(32)
    with pytest.raises(ValueError, match="1 of the 9 BatchNorm containers"):
        m.train()(torch.zeros(2, 1, 256))
    assert fake.calls == []


def test_mixed_groups_raise(fake, world):
    m = converted()
    m.middle[1].process_group = object()
    with pytest.raises(ValueError, match="different process groups"):
        m.train()(torch.zeros(2, 1, 256))
    assert fake.calls == []


def test_reducer_exception_is_reraised_and_the_hook_removed(fake, world):
    class Boom(Exception):
        pass

    m = Model(4, 8).train()

    def bad(buf):
        raise Boom("reducer failed")
    m._bn_allreduce = bad
    with pytest.raises(Boom):
        m(torch.zeros(2, 1, 256))
    assert fake.calls == [("set", True, 65), ("forward_ex", 2, 0), ("hook", 9, 1), ("set", False, 0)]
