"""Eval-mode autograd surface of the drop-in Model, CPU only: the eval_autograd keyword, which eval forwards record a graph,
and the composite path (train_backend="torch") in eval mode against the float64 golden step."""
import os

import numpy as np
import pytest
import torch

from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model


def make_pair(B, T, seed):
    g = np.random.Generator(np.random.PCG64(seed))
    clean = (0.1 * g.standard_normal((B, 1, T))).astype(np.float32)
    noisy = (clean + 0.05 * g.standard_normal((B, 1, T))).astype(np.float32)
    return noisy, clean


def rel_err(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("value", ["input", "always", "off"])
def test_eval_autograd_values_and_state_dict(value):
    m = Model(4, 8, eval_autograd=value)
    assert m.eval_autograd == value
    ref = Model(4, 8)
    assert list(m.state_dict()) == list(ref.state_dict())
    assert not any("eval_autograd" in k for k in m.state_dict())


@pytest.mark.parametrize("value", ["", "on", "Input", None, True])
def test_eval_autograd_rejects_other_values(value):
    with pytest.raises(ValueError, match="eval_autograd"):
        Model(4, 8, eval_autograd=value)


def test_torch_backend_eval_mode_gradients_vs_golden(golden_dir):
    """train_backend="torch", model.eval(), x.requires_grad: the composite path with eval-mode BatchNorm in fp32 on the CPU
    against the float64 reference step; dx and every gradient within 1e-4 of its largest entry."""
    g = np.load(os.path.join(golden_dir, "autograd_small_n4_c8.npz"))
    n, ci, B, T = int(g["n_layers"]), int(g["channels_interval"]), int(g["B"]), int(g["T"])
    st = wo.make_state(n, ci, seed=int(g["state_seed"]))
    noisy, clean = make_pair(B, T, int(g["pair_seed"]))
    m = Model(n, ci, train_backend="torch")
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    m.eval()
    x = torch.from_numpy(noisy).requires_grad_(True)
    y = m(x)
    assert y.grad_fn is not None
    loss = torch.nn.MSELoss()(torch.from_numpy(clean), y)
    loss.backward()
    assert abs(float(loss.detach()) - float(g["eval:loss"])) <= 1e-5 * float(g["eval:loss"])
    errs = {k: rel_err(p.grad.numpy(), g["eval:grad:" + k]) for k, p in m.named_parameters()}
    errs["x"] = rel_err(x.grad.numpy(), g["eval:dx"])
    worst = max(errs.items(), key=lambda kv: kv[1])
    print(f"torch backend, eval mode, CPU fp32: worst rel err {worst[1]:.2e} ({worst[0]}), dx {errs['x']:.2e}")
    assert worst[1] <= 1e-4, worst
    for k, v in m.state_dict().items():
        if "running_" in k:
            assert np.array_equal(v.numpy(), st[k]), k
        elif k.endswith("num_batches_tracked"):
            assert int(v) == 0, k


def _count_native(monkeypatch):
    calls = []

    def fake(self, x):
        calls.append(x.shape)
        return torch.zeros_like(x)

    monkeypatch.setattr(Model, "_forward_native", fake)
    return calls


@pytest.mark.parametrize("backend", ["native", "torch", "none"])
@pytest.mark.parametrize("eval_autograd", ["input", "always", "off"])
def test_eval_forward_without_a_graph_request_goes_through_forward_native(monkeypatch, backend, eval_autograd):
    """A plain input in eval mode takes the inference path (what tests/test_boundary_callers.py patches), also with grad mode
    on and parameters requiring grad, except that "always" with a backend that can record asks for a graph."""
    calls = _count_native(monkeypatch)
    m = Model(4, 8, train_backend=backend, eval_autograd=eval_autograd).eval()
    x = torch.zeros(2, 1, 256)
    with torch.no_grad():
        m(x)
    assert len(calls) == 1
    m.requires_grad_(False)
    m(x)
    assert len(calls) == 2
    m.requires_grad_(True)
    records = eval_autograd == "always" and backend != "none"
    if records and backend == "native":
        with pytest.raises(RuntimeError, match="no CPU fallback"):    # the native training kernels: CUDA only
            m(x)
        assert len(calls) == 2
        return
    y = m(x)
    assert len(calls) == (2 if records else 3)
    if backend == "torch":
        assert (y.grad_fn is not None) == records


@pytest.mark.parametrize("case", ["off", "no_grad", "backend_none", "empty_batch"])
def test_input_requiring_grad_without_a_graph(monkeypatch, case):
    """Cases that keep today's detached eval forward although the input requires grad."""
    calls = _count_native(monkeypatch)
    m = Model(4, 8, train_backend="none" if case == "backend_none" else "torch",
              eval_autograd="off" if case == "off" else "input").eval()
    x = torch.zeros(0 if case == "empty_batch" else 2, 1, 256, requires_grad=True)
    with torch.set_grad_enabled(case != "no_grad"):
        m(x)
    assert len(calls) == 1


def test_input_requiring_grad_records_a_graph_on_the_torch_backend(monkeypatch):
    calls = _count_native(monkeypatch)
    m = Model(4, 8, train_backend="torch").eval()
    x = torch.randn(2, 1, 256, requires_grad=True)
    m(x).sum().backward()
    assert not calls
    assert x.grad is not None and x.grad.shape == x.shape


@pytest.mark.parametrize("n,ci", [(12, 24), (4, 8)])
def test_one_value_per_channel_raises_like_batchnorm(n, ci):
    """Training mode, B = 1, T = 2^n_layers: the middle block sees one value per channel and torch.nn.BatchNorm1d raises its
    ValueError. The native backend raises the same error before it needs a GPU; eval mode (running statistics) accepts it."""
    x = torch.zeros(1, 1, 1 << n)
    msgs = []
    for backend in ("torch", "native"):
        m = Model(n, ci, train_backend=backend).train()
        with pytest.raises(ValueError, match="Expected more than 1 value per channel when training") as e:
            m(x)
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1]
    m = Model(n, ci, train_backend="torch").eval()
    assert m(x.clone().requires_grad_(True)).shape == x.shape
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        Model(n, ci).train()(torch.zeros(1, 1, 2 << n))           # two values per channel: on to the device check
