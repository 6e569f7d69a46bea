"""The ping-pong form of the last decoder block (csrc/wunet_tc_pp.cuh) gives the bits of the recorded form.

At 12 levels x 24 base filters the last decoder block (24, fused with the head) keeps its weights in shared memory and runs the
ping-pong kernel: each consumer warpgroup owns every other tile of its CTA. The same block with ``res=0`` (weights streamed from
L2) runs the recorded conv_tc_kernel, whose K loop and epilogue arithmetic are the same, so the block's output and the network
output must be equal bit for bit. The SM counts give CTAs an even or odd number of tiles, or a single one (the second warpgroup has
none): B = 1 has 128 tiles per block, B = 3 has 384. bf16 and fp16 (the fp16 twins of both forms)."""
import numpy as np
import pytest
import torch

from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model, _lib

pytestmark = [pytest.mark.gpu]

N, CI, T = 12, 24, 16384
BLOCK = 24
STREAMED = "%d:res=0" % BLOCK
# (B, WUNET_TC_SMS): tiles per CTA 128 | 18-19 | 1-2 | 1, and 384 | 54-55 | 3-4
CASES = [(1, 1), (1, 7), (1, 100), (1, 128), (3, 1), (3, 7), (3, 100)]
KNOBS = ("WUNET_TC_SMS", "WUNET_TC_OVR", "WUNET_TC_GEMM", "WUNET_TC_STORE_LAST", "WUNET_TC_PAIR", "WUNET_TC_ENC0",
         "WUNET_TC_ENC0V", "WUNET_TC_MERGE")


def run(precision, B, monkeypatch, ovr=None):
    if ovr is None:
        monkeypatch.delenv("WUNET_TC_OVR", raising=False)
    else:
        monkeypatch.setenv("WUNET_TC_OVR", ovr)
    m = Model(N, CI, precision=precision)
    st = wo.make_state(N, CI, seed=3)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    m = m.to("cuda:0").eval()
    x = torch.from_numpy(wo.make_input(B, T, seed=40 + B)).to("cuda:0")
    with torch.no_grad():
        y = m(x)
    level = m.read_level(BLOCK, B, T)
    torch.cuda.synchronize()
    m._release()
    return y, level


@pytest.mark.parametrize("precision", ("bf16", "fp16"))
@pytest.mark.parametrize("B,sms", CASES)
def test_pingpong_block_gives_the_recorded_bits(B, sms, precision, monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")
    monkeypatch.setenv("WUNET_TC_SMS", str(sms))
    d = _lib.debug_plan(N, CI, B, T, BLOCK, sms, precision)   # the default plan runs the ping-pong form, the override the recorded one
    assert d["resident"] == 1 and d["nsplit"] == 1 and d["small"] == 0 and d["packed"] == 0 and d["Nh"] <= 80, d
    y_pp, lv_pp = run(precision, B, monkeypatch)
    y_ref, lv_ref = run(precision, B, monkeypatch, ovr=STREAMED)
    assert torch.equal(lv_pp, lv_ref), "block output differs from the recorded form"
    assert torch.equal(y_pp, y_ref), "output differs from the recorded form"
