"""Wide channel plans (channels_interval 40 .. 64) on the tensor cores, on an H100: every level and the output against the C
oracle at all three tensor-core precisions, the persistent regime against precision="fp32" on the same GPU, the same bits
from every host entry point, and a model trained natively at a wide width that then runs eval at the default precision.

Bars: the ones the existing parity tests use for each precision (test_parity_gpu.py: fp32_tc 1e-4, bf16 8e-3 of a level's
largest magnitude and 2e-3 on the output; test_fp16_gpu.py: fp16 3e-4, to which a level adds the half-ulp rounding of its own
fp16 store, 2^-11 of its magnitude, since these levels exceed 1). A wider plan sums more products per output (K = ci x
taps per segment grows with ci), but the error of a 16-bit operand is a rounding error per product, relative to that product;
summed with random signs it grows with the square root of K while the level's magnitude, set by BatchNorm, does not. ci = 64
has K (64 / 24)^(1/2) = 1.6 times the reference's error for the same operand rounding, inside the margin of every bar above
(measured at 24: bf16 0.3-0.5 % of 0.8 %, fp16 7e-5 of 3e-4, fp32_tc 1e-6 of 1e-4), so the bars are not widened."""
import numpy as np
import pytest
import torch

from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model
from wave_u_net_for_speech_enhancement_b200.enhance import enhance_waveforms, frame_clips, unframe_clips

pytestmark = [pytest.mark.gpu]

TC_PRECISIONS = ["fp32_tc", "bf16", "fp16"]
SWITCHES = ("WUNET_TC_SMS", "WUNET_TC_OVR", "WUNET_TC_GEMM", "WUNET_TC_STORE_LAST", "WUNET_TC_ENC0", "WUNET_TC_PAIR",
            "WUNET_TC_MERGE")
OUT_TOL = {"fp32_tc": 1e-4, "bf16": 2e-3, "fp16": 3e-4}


def level_ok(prec, err, ref_max):
    if prec == "fp32_tc":
        return err <= 1e-4 * max(1.0, ref_max)
    if prec == "bf16":
        return err <= 8e-3 * ref_max
    # fp16: the same 3e-4 for what a level inherits, plus the rounding of its own fp16 store, half an ulp = 2^-11 of its
    # magnitude (4.9e-4 at a level that reaches 1.47; test_fp16_gpu.py's small levels did not meet it)
    return err <= 3e-4 * max(1.0, ref_max) + 2.0 ** -11 * ref_max


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)


def make_model(n, ci, st, precision):
    m = Model(n, ci, precision=precision)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    return m.to("cuda:0").eval()


def run(m, x):
    with torch.no_grad():
        return m(torch.from_numpy(np.ascontiguousarray(x)).cuda())


@pytest.mark.parametrize("prec", TC_PRECISIONS)
@pytest.mark.parametrize("n,ci,B,T", [(5, 40, 3, 4096), (5, 48, 2, 4096), (6, 64, 3, 2048), (12, 48, 2, 16384)])
def test_levels_and_output_vs_oracle(n, ci, B, T, prec, monkeypatch):
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")
    st = wo.make_state(n, ci, seed=ci + n)
    x = wo.make_input(B, T, seed=7 * ci + B)
    x[-1, 0, 0] += 0.9                                  # both frame edges: zero padding and the ends of the upsampling
    x[-1, 0, T - 1] -= 0.9
    want_y, want = wo.COracle(n, ci).forward(st, x, return_levels=True)
    m = make_model(n, ci, st, prec)
    y = run(m, x).cpu().numpy()
    errs = []
    for i in range(2 * n + 1):
        lv = m.read_level(i, B, T).cpu().numpy()
        ref_max = float(np.abs(want[i]).max())
        err = float(np.abs(lv - want[i]).max())
        errs.append(err / max(1.0, ref_max))
        assert level_ok(prec, err, ref_max), (i, err, ref_max)
    yerr = float(np.abs(y - want_y).max())
    print(f"{prec} n={n} ci={ci}: worst level error (relative to max(1, |level|)) {max(errs):.2e}, output {yerr:.2e}")
    assert yerr <= OUT_TOL[prec], yerr
    assert m.last_launch_count() == 2 * n + 1
    m._release()
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "0")   # the benchmarked form: head fused, last block not stored
    assert torch.equal(run(make_model(n, ci, st, prec), x).cpu(), torch.from_numpy(y))


@pytest.mark.parametrize("B", [256, 257])
@pytest.mark.parametrize("n,ci", [(12, 48), (12, 64)])
def test_persistent_regime_vs_fp32(n, ci, B):
    """Batches that fill every SM several times over (257: one frame past a multiple of the SM count), each tensor-core precision
    against the CUDA-core fp32 path on the same weights."""
    T = 16384
    st = wo.make_state(n, ci, seed=5)
    x = wo.make_input(B, T, seed=B)
    m = make_model(n, ci, st, "fp32")
    ref = run(m, x)
    m._release()
    for prec in TC_PRECISIONS:
        m = make_model(n, ci, st, prec)
        y = run(m, x)
        m._release()
        err = float((y - ref).abs().max())
        print(f"n={n} ci={ci} B={B} {prec}: max-abs vs fp32 {err:.2e}")
        assert torch.isfinite(y).all() and err <= OUT_TOL[prec], (prec, err)
        del y
    torch.cuda.empty_cache()


@pytest.mark.parametrize("prec", TC_PRECISIONS)
def test_entry_points_agree_bit_for_bit(prec):
    n, ci, T = 8, 48, 4096
    st = wo.make_state(n, ci, seed=9)
    m = make_model(n, ci, st, prec)
    x = wo.make_input(8, T, seed=10)
    y = run(m, x).cpu()
    assert torch.equal(run(m, x).cpu(), y), "a repeated forward differs"
    xh = torch.from_numpy(x).pin_memory()
    assert torch.equal(m.forward_host(xh), y), "forward_host differs from forward"
    outs = list(m.forward_host_stream([xh[:4].contiguous(), xh[4:].contiguous()]))
    for half, o in zip((x[:4], x[4:]), outs):
        assert torch.equal(run(m, half).cpu(), o), "forward_host_stream differs from forward"
    rng = np.random.default_rng(7)
    clips = [(0.1 * rng.standard_normal(L)).astype(np.float32) for L in (4 * T, 3 * T + 1000)]
    got = enhance_waveforms(m, clips, sample_length=T, batch_frames=4)
    frames, index = frame_clips(clips, T, round_to=4)
    with torch.no_grad():
        yf = torch.cat([m(frames[i:i + 4].cuda()).cpu() for i in range(0, frames.shape[0], 4)])
    assert all(np.array_equal(a, b) for a, b in zip(got, unframe_clips(yf, index, True))), "enhance_waveforms differs"


def test_trained_wide_model_runs_eval_at_the_default_precision():
    """A config with channels_interval = 48 trains with the native bf16 step; the validation forward that follows (eval mode,
    no_grad, default precision) used to be refused."""
    torch.manual_seed(0)
    n, ci, T = 12, 48, 16384
    model = Model(n, ci, train_precision="bf16").cuda()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    mix = torch.from_numpy(wo.make_input(4, T, seed=1)).cuda()
    clean = 0.5 * mix
    model.train()
    for _ in range(2):
        opt.zero_grad()
        loss = torch.nn.functional.mse_loss(model(mix), clean)
        loss.backward()
        opt.step()
    model.eval()
    assert model.precision == "fp32_tc"
    with torch.no_grad():
        y = model(mix)
    assert torch.isfinite(y).all()
    ref = Model(n, ci, precision="fp32")
    ref.load_state_dict(model.state_dict())
    ref = ref.cuda().eval()
    with torch.no_grad():
        err = float((y - ref(mix)).abs().max())
    print(f"trained n=12 ci=48: fp32_tc vs fp32 max-abs {err:.2e}")
    assert err <= OUT_TOL["fp32_tc"], err
