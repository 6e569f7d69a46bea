"""bf16 tensor-core path against its arithmetic model (oracle/wunet_bf16_model.py): level by level, the kernels must
reproduce the model's bf16 values except where the fp32 accumulation order flips a rounding (a one-ulp difference at a
small fraction of the elements). Much sharper than the tolerance against the fp32 oracle (test_parity_gpu.py).

A value may differ from the model's by one bf16 ulp where the fp32 accumulation order flips the final rounding; where the
pre-activation cancels to almost zero the flip is an fp32 rounding error of the SUM (relative to the terms, not the result),
so differences are also accepted up to ABS_FLOOR x the level's largest magnitude."""
import os

import numpy as np
import pytest
import torch

from oracle import wunet_bf16_model as wb
from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model

pytestmark = [pytest.mark.gpu]

ABS_FLOOR = 2.0 ** -11       # of the level's max |value|


def lib_enc0_tc(ci, T):
    """Does the library run the first block on the tensor cores (3 taps over groups of 8 samples, bf16 samples and weights) for
    this shape? Mirrors build_plan: WUNET_TC_ENC0, frames of at least 1024 samples, 8 C <= 256 columns."""
    return os.environ.get("WUNET_TC_ENC0", "0") == "1" and T % 8 == 0 and T // 8 >= 128 and ci % 8 == 0 and 8 * ci <= 256


def ulp_bf16(v):
    """spacing of bf16 numbers at |v| (8 significant bits)"""
    return np.exp2(np.floor(np.log2(np.maximum(np.abs(v), 1e-30))) - 7)


def make_model(n, ci, st, precision):
    m = Model(n, ci, precision=precision)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()})
    return m.to("cuda:0").eval()


def run(m, x, pick=None):
    """Forward of the whole batch x; -> output and the 2n+1 block outputs, as device tensors, of the frames in pick (all: None).
    The levels are sliced on the device: at B = 256 block 0 alone is 400 MB in fp32."""
    B, _, T = x.shape
    idx = None if pick is None else torch.tensor(pick, device="cuda:0")
    with torch.no_grad():
        y = m(torch.from_numpy(x).cuda())
    levels = []
    for i in range(2 * m.n_layers + 1):
        lv = m.read_level(i, B, T)
        levels.append(lv if idx is None else lv.index_select(0, idx))
    return y, levels


# (n, ci, B, T, seed); PICKS: the frames checked against the model (all frames for a batch not listed). The third case has
# batch >= 64: blocks of at most 16 samples (enc5, middle, dec0 there) run the dense GEMM over frames, the decoder among them
# with the interpolation folded into its weights. The last two are the regime the benchmark times: persistent CTAs that run 62 to 249 tiles of the top blocks with
# resident weights, blocks 10-14 on the GEMM with 2 (3) row tiles of 128 frames, blocks 9 and 15 in packed tiles of 3 frames.
# The picked frames hit the packed-tile boundaries (2 | 3, 127 | 128 | 129), both GEMM row tiles, the lone frame 255 in the last
# packed tile at B = 256; at B = 257 the third GEMM row tile holds frame 256 alone and the last packed tile holds 255 and 256.
PICK = [0, 1, 2, 3, 127, 128, 254, 255]
PICKS = {256: PICK, 257: PICK + [256]}
MODEL_CASES = [(4, 8, 3, 256, 11), (12, 24, 2, 16384, 0), (6, 8, 64, 512, 5), (12, 24, 256, 16384, 0), (12, 24, 257, 16384, 0)]
# the B = 256 case must also give the same bits without the last block stored (the benchmarked variant) and planned for this
# SM count (an H100 PCIe)
OTHER_SMS = 114


@pytest.mark.parametrize("n,ci,B,T,seed", MODEL_CASES)
def test_levels_match_the_arithmetic_model(n, ci, B, T, seed, monkeypatch):
    pick = PICKS.get(B)
    for k in ("WUNET_TC_SMS", "WUNET_TC_OVR", "WUNET_TC_GEMM"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")               # materialise the last decoder block too
    st = wo.make_state(n, ci, seed=seed)
    x = wo.make_input(B, T, seed=seed + 100)
    m = make_model(n, ci, st, "bf16")
    y_dev, lv_dev = run(m, x, pick)
    xs = x if pick is None else x[pick]
    y = (y_dev if pick is None else y_dev[pick]).cpu().numpy()
    got_levels = [lv.cpu().numpy() for lv in lv_dev]
    # every block of the model is evaluated on the GPU's own outputs of the blocks before it: a rounding flip stays local. The
    # library takes the dense GEMM from the size of the whole batch, not of the subset
    want_y, want = wb.forward_bf16_model(st, xs, n, ci, return_levels=True, forced=got_levels[:2 * n], dense_bottom=B >= 64,
                                         enc0_tc=lib_enc0_tc(ci, T))
    report = []
    for i in range(2 * n + 1):
        got = got_levels[i]
        ref = want[i] if i < 2 * n else want[i].astype(np.float32)
        if i == 2 * n:                                           # the stored copy of the last block is rounded to bf16
            ref = torch.from_numpy(ref).to(torch.bfloat16).float().numpy()
        diff = np.abs(got - ref)
        frac_equal = float((diff == 0).mean())
        excess = float((diff - np.maximum(2.0 * ulp_bf16(ref), ABS_FLOOR * np.abs(ref).max())).max())
        report.append((i, round(frac_equal, 5), float(diff.max()), excess))
    yerr = float(np.abs(y - want_y).max())
    print("bf16 model (teacher-forced) vs kernels: (block, fraction bit-equal, max abs diff, excess over bound)")
    for r in report:
        print("   ", r)
    print("    output max-abs diff", yerr)
    assert all(r[1] >= 0.995 for r in report), report
    assert all(r[3] <= 0.0 for r in report), report
    assert yerr <= 2e-5, (yerr, report)
    if B != 256:
        return
    # the same bits, over the whole batch, from the benchmarked variant (last block not stored) and from another SM count
    y_all, lv_all = run(m, x)
    m._release()
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "0")
    m0 = make_model(n, ci, st, "bf16")
    with torch.no_grad():
        assert torch.equal(m0(torch.from_numpy(x).cuda()), y_all), "WUNET_TC_STORE_LAST=0 changes the output"
    m0._release()
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")
    monkeypatch.setenv("WUNET_TC_SMS", str(OTHER_SMS))
    y2, lv2 = run(make_model(n, ci, st, "bf16"), x)
    assert [i for i in range(2 * n + 1) if not torch.equal(lv2[i], lv_all[i])] == [], f"WUNET_TC_SMS={OTHER_SMS}: blocks differ"
    assert torch.equal(y2, y_all), f"WUNET_TC_SMS={OTHER_SMS}: output differs"


FP32_TC_CASE = (12, 24, 256, 16384, 0)


def test_fp32_tc_levels_at_batch_256(monkeypatch):
    """fp32_tc, the Model default, in the persistent regime: every block of the picked frames against the fp32 oracle."""
    n, ci, B, T, seed = FP32_TC_CASE
    pick = PICKS[B]
    for k in ("WUNET_TC_SMS", "WUNET_TC_OVR", "WUNET_TC_GEMM"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")
    st = wo.make_state(n, ci, seed=seed)
    x = wo.make_input(B, T, seed=seed + 100)
    y, got = run(make_model(n, ci, st, "fp32_tc"), x, pick)
    want_y, want = wo.COracle(n, ci).forward(st, x[pick], return_levels=True)
    errs = [float(np.abs(g.cpu().numpy() - w).max()) for g, w in zip(got, want)]
    yerr = float(np.abs(y[pick].cpu().numpy() - want_y).max())
    print("fp32_tc B=256 per-block max-abs errors " + " ".join("%.1e" % e for e in errs) + " | output %.1e" % yerr)
    assert max(errs) <= 1e-4, errs
    assert yerr <= 1e-4, yerr
