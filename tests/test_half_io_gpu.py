"""Half models on an H100: ``model.half()`` / ``model.to(torch.bfloat16)`` take and return 16-bit tensors, and compute exactly
what the float32 model computes on the widened parameters and samples, rounded once at the output:
``half_model(x16) == float_model(x16.float()).to(x16.dtype)`` bit for bit, at every precision, through every entry point."""
import numpy as np
import pytest
import torch

from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model
from wave_u_net_for_speech_enhancement_b200.enhance import enhance_waveforms

pytestmark = [pytest.mark.gpu]

DEV = "cuda:0"
DTYPES = [torch.float16, torch.bfloat16]
PRECISIONS = ["fp32", "fp32_tc", "bf16", "fp16"]
PLANS = [(12, 24), (12, 48), (4, 8)]
SHAPES = [(1, 16384), (2, 16384), (256, 16384), (257, 16384), (2, 4096)]


def rounded_state(n, ci, dtype, seed=0):
    """the oracle's random state with every tensor rounded to `dtype` (so that the float32 model holds the same values)"""
    st = wo.make_state(n, ci, seed=seed)
    return {k: torch.from_numpy(np.asarray(v)).to(dtype).float() if np.asarray(v).dtype.kind == "f" else torch.from_numpy(np.asarray(v))
            for k, v in st.items()}


def models(n, ci, precision, dtype, seed=0):
    """(float32 model, the same model converted to dtype), both on the GPU in eval mode"""
    sd = rounded_state(n, ci, dtype, seed)
    m32 = Model(n, ci, precision=precision)
    m32.load_state_dict(sd, strict=True)
    m16 = Model(n, ci, precision=precision)
    m16.load_state_dict(sd, strict=True)
    return m32.to(DEV).eval(), m16.to(DEV).to(dtype).eval()


def x16(B, T, dtype, seed=1234):
    return torch.from_numpy(wo.make_input(B, T, seed=seed)).to(dtype)


def mismatches(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape
    return int((a.view(torch.int16) != b.view(torch.int16)).sum())


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("plan", PLANS, ids=[f"n{n}c{c}" for n, c in PLANS])
def test_half_model_is_the_float_model_rounded_once(plan, precision, dtype):
    n, ci = plan
    m32, m16 = models(n, ci, precision, dtype)
    bad = {}
    with torch.no_grad():
        for B, T in SHAPES:
            x = x16(B, T, dtype).to(DEV)
            y = m16(x)
            assert y.dtype == dtype and y.shape == x.shape
            want = m32(x.float()).to(dtype)
            d = mismatches(y, want)
            if d:
                bad[(B, T)] = d
    assert not bad, f"differing elements per (B, T): {bad}"


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("precision", ["fp32", "bf16", "fp32_tc"])
def test_every_entry_point_agrees(precision, dtype):
    m32, m16 = models(12, 24, precision, dtype)
    B, T = 8, 16384
    x = x16(B, T, dtype)
    with torch.no_grad():
        dev = m16(x.to(DEV)).cpu()
        host = m16.forward_host(x.pin_memory())
        batches = [x[:4].pin_memory(), x[4:].pin_memory()]
        stream = torch.cat([o.clone() for o in m16.forward_host_stream(batches)])
        want = m32(x.float().to(DEV)).to(dtype).cpu()
    assert host.dtype == stream.dtype == dtype
    assert mismatches(dev, want) == 0
    assert mismatches(host, dev) == 0
    assert mismatches(stream, dev) == 0


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_enhance_waveforms_on_a_half_model(dtype):
    m32, m16 = models(12, 24, "bf16", dtype)
    rng = np.random.default_rng(5)
    lengths = [16384 * 3 + 17, 900, 16384]
    clips_f = [rng.uniform(-0.5, 0.5, n).astype(np.float32) for n in lengths]
    clips_i = [rng.integers(-32768, 32767, n, dtype=np.int16) for n in lengths]
    for clips in (clips_f, clips_i):
        got = enhance_waveforms(m16, clips, batch_frames=4)
        assert [g.dtype for g in got] == [np.float32] * 3 and [len(g) for g in got] == lengths
        for g, c in zip(got, clips):
            # the reference loop on the float32 model, with the frame's samples rounded once to the I/O dtype
            s = torch.from_numpy(c.astype(np.float32) / (32768.0 if c.dtype == np.int16 else 1.0))
            nf = -(-len(c) // 16384)
            frames = torch.zeros(nf * 16384)
            frames[:len(c)] = s
            frames = frames.view(nf, 1, 16384).to(dtype)
            with torch.no_grad():
                one = m16(frames.to(DEV)).cpu()
                want = m32(frames.float().to(DEV)).to(dtype).cpu()
            assert mismatches(one, want) == 0
            assert np.array_equal(g, one.float().view(-1).numpy()[:len(c)])


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_refusals(dtype):
    m32, m16 = models(4, 8, "bf16", dtype)
    x = x16(2, 256, dtype).to(DEV)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="input"):
            m16(x.float())                                   # float32 input, half model
        with pytest.raises(RuntimeError, match="input"):
            m32(x)                                           # 16-bit input, float32 model
    m16.train()
    with pytest.raises(RuntimeError, match="train_precision"):
        m16(x)
    m16.eval()
    with pytest.raises(RuntimeError, match="train_precision"):
        m16(x.clone().requires_grad_(True))                  # an eval forward that records a graph
    mixed = Model(4, 8, precision="bf16").to(DEV).to(dtype).eval()
    mixed.out[0].weight.data = mixed.out[0].weight.data.float()
    with torch.no_grad(), pytest.raises(RuntimeError, match="float32"):
        mixed(x.float())


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_half_checkpoint_and_the_shared_context(dtype):
    m32, m16 = models(12, 24, "bf16", dtype)
    x = x16(2, 16384, dtype).to(DEV)
    with torch.no_grad():
        y16 = m16(x)
        sd = m16.state_dict()
        assert all(v.dtype in (dtype, torch.int64) for v in sd.values())
        other = Model(12, 24, precision="bf16").to(dtype)
        other.load_state_dict(sd, strict=True)
        assert mismatches(other.to(DEV).eval()(x), y16) == 0
        # one model, one native context: float32, then half, then float32 again
        y32 = m32(x.float())
        m32.to(dtype)
        assert mismatches(m32(x), y16) == 0
        m32.float()
        assert torch.equal(m32(x.float()), y32)
