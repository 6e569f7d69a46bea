"""Deterministic mode of the native training step, host side (no GPU): the public flag, and how the Python layer selects it
from PyTorch's two determinism switches. The library calls are recorded through a fake binding; the workspace sizes
themselves need a device context and are checked in test_train_deterministic_gpu.py."""
import contextlib
import inspect
import os
import re
import types

import pytest
import torch

from wave_u_net_for_speech_enhancement_b200 import Model, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header():
    return open(os.path.join(ROOT, "include", "wunet_b200.h")).read()


def test_flag_value_in_header_and_binding():
    flags = dict(re.findall(r"#define\s+(WUNET_TRAIN_[A-Z_]+)\s+(\d+)", header()))
    assert flags == {"WUNET_TRAIN_FROZEN_BN": "1", "WUNET_TRAIN_NO_PARAM_GRADS": "2", "WUNET_TRAIN_DETERMINISTIC": "16"}
    assert _lib.TRAIN_DETERMINISTIC == 16
    assert "wunet_train_workspace_bytes_ex" in _lib.EXPORTED_SYMBOLS
    assert re.search(r"size_t\s+wunet_train_workspace_bytes_ex\s*\(\s*const wunet_ctx \*ctx,\s*int B,\s*int T,\s*int precision,"
                     r"\s*int flags\s*\)", header())


def test_constructor_surface_is_unchanged():
    params = inspect.signature(Model.__init__).parameters
    assert [(p.name, p.default) for p in list(params.values())[1:]] == [
        ("n_layers", 12), ("channels_interval", 24), ("precision", "fp32_tc"), ("train_backend", "native"),
        ("data_parallel", "auto"), ("train_precision", "fp32"), ("eval_autograd", "input")]


class FakeLib:
    """Records the flags of the workspace query and of the forward; sizes the workspace at 64 bytes."""

    def __init__(self):
        self.calls = []

    def wunet_train_workspace_bytes_ex(self, c, B, T, prec, flags):
        self.calls.append(("workspace_bytes_ex", B, T, prec, flags))
        return 64

    def wunet_train_forward_ex(self, c, x, y, B, T, *rest):
        self.calls.append(("forward_ex", B, T, rest[-2], rest[-1]))
        return 0


@pytest.fixture
def fake_native(monkeypatch):
    """Model.forward on the CPU against FakeLib: the device plumbing is stubbed and inputs pass the CUDA check; everything
    from the switch lookup in Model.forward to the C calls of the autograd Function is the real code."""
    lib = FakeLib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda d=None: types.SimpleNamespace(cuda_stream=0))
    monkeypatch.setattr(Model, "_context", lambda self, d: None)
    return lib


@contextlib.contextmanager
def switches(cudnn, algorithms):
    saved = (torch.backends.cudnn.deterministic, torch.are_deterministic_algorithms_enabled())
    torch.backends.cudnn.deterministic = cudnn
    torch.use_deterministic_algorithms(algorithms)
    try:
        yield
    finally:
        torch.backends.cudnn.deterministic = saved[0]
        torch.use_deterministic_algorithms(saved[1])


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("cudnn, algorithms", [(False, False), (True, False), (False, True), (True, True)])
def test_either_torch_switch_selects_deterministic_mode(fake_native, mode, prec, cudnn, algorithms):
    """Each switch alone sets WUNET_TRAIN_DETERMINISTIC in the workspace query and in the forward; with both off the flags
    are exactly those of a step without deterministic mode (0 in training, WUNET_TRAIN_FROZEN_BN in an eval forward that
    records a graph)."""
    m = Model(4, 8, train_precision=prec).train(mode == "train")
    x = torch.zeros(2, 1, 256, requires_grad=(mode == "eval"))
    with switches(cudnn, algorithms):
        y = m(x)
    assert y.shape == x.shape and y.grad_fn is not None
    base = 0 if mode == "train" else _lib.TRAIN_FROZEN_BN
    want = base | (_lib.TRAIN_DETERMINISTIC if (cudnn or algorithms) else 0)
    p = _lib.PRECISIONS[prec]
    assert fake_native.calls == [("workspace_bytes_ex", 2, 256, p, want), ("forward_ex", 2, 256, p, want)]


def test_switches_are_read_at_each_call(fake_native):
    """The mode follows the switches as they are when the forward runs, not when the model was built."""
    m = Model(4, 8).train()
    with switches(True, False):
        m(torch.zeros(2, 1, 256))
    m(torch.zeros(2, 1, 256))
    assert [c[-1] for c in fake_native.calls if c[0] == "forward_ex"] == [_lib.TRAIN_DETERMINISTIC, 0]
