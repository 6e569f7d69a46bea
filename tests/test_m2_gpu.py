"""The 256-row form of the streamed-weight blocks (csrc/wunet_tc_m2.cuh) gives the bits of the 128-row form.

Each selected block runs its K loop per accumulator in conv_tc_kernel's order (chunk, tap, K16 step; only the weight stages
group the taps differently) and the same epilogue arithmetic, so its output and the network output must be equal bit for bit to
the same forward with WUNET_TC_M2=0, which runs every block in conv_tc_kernel. bf16 and fp16, at the benchmark shape, under SM
counts that give CTAs one, two, an odd or an even number of units and an uneven last round, on a wide channel plan, and on
resident blocks whose weights an override streams."""
import numpy as np
import pytest
import torch

from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model, _lib

pytestmark = [pytest.mark.gpu]

N, T = 12, 16384
KNOBS = ("WUNET_TC_SMS", "WUNET_TC_OVR", "WUNET_TC_GEMM", "WUNET_TC_STORE_LAST", "WUNET_TC_PAIR", "WUNET_TC_ENC0",
         "WUNET_TC_ENC0V", "WUNET_TC_MERGE", "WUNET_TC_M2")


def selected(ci, B, sms, precision):
    return [i for i in range(1, 2 * N + 1) if _lib.debug_plan_m2(N, ci, B, T, i, sms, precision)["selected"]]


def run(precision, ci, B, blocks, monkeypatch, on):
    monkeypatch.setenv("WUNET_TC_M2", "1" if on else "0")      # read when the library creates the model's tensor-core state
    m = Model(N, ci, precision=precision)
    st = wo.make_state(N, ci, seed=3)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    m = m.to("cuda:0").eval()
    x = torch.from_numpy(wo.make_input(B, T, seed=40 + B)).to("cuda:0")
    with torch.no_grad():
        y = m(x)
    levels = {i: m.read_level(i, B, T) for i in blocks}
    torch.cuda.synchronize()
    m._release()
    return y, levels


def check(precision, ci, B, sms, monkeypatch, ovr=None, want=None):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    if ovr is not None:
        monkeypatch.setenv("WUNET_TC_OVR", ovr)
    if sms is not None:
        monkeypatch.setenv("WUNET_TC_SMS", str(sms))
    num_sms = sms if sms is not None else torch.cuda.get_device_properties(0).multi_processor_count
    blocks = selected(ci, B, num_sms, precision)
    if want is not None:
        assert set(want) <= set(blocks), (want, blocks)
    assert blocks, "no block runs the 256-row form here"
    y_on, lv_on = run(precision, ci, B, blocks, monkeypatch, True)
    y_off, lv_off = run(precision, ci, B, blocks, monkeypatch, False)
    for i in blocks:
        assert torch.equal(lv_on[i], lv_off[i]), "block %d differs from the 128-row form" % i
    assert torch.equal(y_on, y_off), "output differs from the 128-row form"


@pytest.mark.parametrize("precision", ("bf16", "fp16"))
def test_benchmark_shape_gives_the_recorded_bits(precision, monkeypatch):
    check(precision, 24, 256, None, monkeypatch, want=[3, 5, 6, 18, 19, 21])


# B = 8: units per block 64 (enc3, dec8), 32 (enc5, dec6), 16 (enc6, dec5). SM counts 1 (one CTA: all units), 2 (even),
# 7 (odd, uneven last rounds: 64 = 9 x 7 + 1), 16 (one unit per CTA in enc6 / dec5), 32 (one in enc5 / dec6; two in enc3)
@pytest.mark.parametrize("precision", ("bf16", "fp16"))
@pytest.mark.parametrize("sms", (1, 2, 7, 16, 32))
def test_unit_distributions_give_the_recorded_bits(precision, sms, monkeypatch):
    check(precision, 24, 8, sms, monkeypatch)


@pytest.mark.parametrize("precision", ("bf16", "fp16"))
def test_wide_plan_gives_the_recorded_bits(precision, monkeypatch):
    check(precision, 48, 4, 7, monkeypatch)


@pytest.mark.parametrize("precision", ("bf16", "fp16"))
def test_streamed_resident_blocks_give_the_recorded_bits(precision, monkeypatch):
    # enc2 and dec9 keep their weights in shared memory by default; streamed, the rule selects them
    check(precision, 24, 8, 7, monkeypatch, ovr="2:res=0;22:res=0", want=[2, 22])
