"""When the decoder producers prefetch: by default each thread issues the global loads of its first item of an upsampled chunk
when the K loop reaches that chunk, just before it waits for the chunk's operand stage; ``WUNET_TC_PFLATE=0`` issues them
right after the previous upsampled chunk's hand-off instead. Both load the same previous-level rows into the same registers
and interpolate them in the same order, so every block output (``WUNET_TC_STORE_LAST=1``) and the network output must be
bit-identical."""
import numpy as np
import pytest
import torch

from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model

pytestmark = [pytest.mark.gpu]

KNOBS = ("WUNET_TC_SMS", "WUNET_TC_OVR", "WUNET_TC_GEMM", "WUNET_TC_PAIR", "WUNET_TC_ENC0", "WUNET_TC_ENC0V", "WUNET_TC_MERGE",
         "WUNET_TC_PFLATE")


def run_levels(n, ci, B, T):
    """Fresh model (the library reads WUNET_TC_PFLATE / WUNET_TC_STORE_LAST when it creates the model's state), one seeded bf16
    forward: the output and all 2n + 1 block outputs."""
    m = Model(n, ci, precision="bf16")
    st = wo.make_state(n, ci, seed=0)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    m = m.to("cuda:0").eval()
    x = torch.from_numpy(wo.make_input(B, T, seed=500 + B + T)).to("cuda:0")
    with torch.no_grad():
        y = m(x)
    lv = [m.read_level(i, B, T) for i in range(2 * n + 1)]
    torch.cuda.synchronize()
    m._release()
    return y, lv


# (n_layers, channels_interval, B, T, WUNET_TC_SMS or None): the benchmark's blocks at a small batch, a batch whose tiles do
# not divide evenly over the persistent grid, a grid of 7 SMs (many tiles per CTA), and the small configuration
CASES = [(12, 24, 5, 16384, None), (12, 24, 33, 4096, None), (12, 24, 5, 16384, 7), (4, 8, 3, 256, None)]


@pytest.mark.parametrize("n,ci,B,T,sms", CASES)
def test_prefetch_point_does_not_change_the_bits(n, ci, B, T, sms, monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")
    if sms is not None:
        monkeypatch.setenv("WUNET_TC_SMS", str(sms))
    y0, l0 = run_levels(n, ci, B, T)
    monkeypatch.setenv("WUNET_TC_PFLATE", "0")
    y1, l1 = run_levels(n, ci, B, T)
    bad = [i for i, (a, b) in enumerate(zip(l0, l1)) if not torch.equal(a, b)]
    assert not bad, f"blocks {bad} differ between the two prefetch points"
    assert torch.equal(y0, y1)
