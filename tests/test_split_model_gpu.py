"""fp32_tc (the Model default: split bf16 precision on the tensor cores) and fp32 (FFMA) inference against their float64
arithmetic model (tests/split_model.py), block by block and teacher-forced: every block is evaluated on the GPU's own outputs
of the blocks before it and held to a bar from its own arithmetic, |s| sum |products| for the K loop and one storage rounding.
A dropped or mis-paired term of one K chunk of one block moves that block by 2-5e-4 of its |s| sum |products|, 16x and more
over its bar, but the network output by as little as 4e-7: the oracle checks at 1e-4 (test_parity_gpu.py) cannot see it.
The file runs in 20-25 s on an H100 80GB HBM3 (700 W).

Per case the log shows, per block, the worst error / bar and the fraction of elements equal to the model's split(fp32(v))
(as hi + lo), then the output's worst error / bar."""
import time
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import pytest
import torch

import split_model as sm
from oracle import wunet_oracle as wo
from test_bf16_model_gpu import PICKS
from wave_u_net_for_speech_enhancement_b200 import Model

pytestmark = [pytest.mark.gpu]

DEV = "cuda:0"
ENV_KNOBS = ("WUNET_TC_SMS", "WUNET_TC_OVR", "WUNET_TC_GEMM", "WUNET_TC_MERGE", "WUNET_TC_PAIR", "WUNET_TC_ENC0V",
             "WUNET_TC_STORE_LAST")


@dataclass(frozen=True)
class Case:
    name: str
    n: int
    ci: int
    B: int
    T: int
    seed: int = 0
    edges: bool = False                 # frame 0: impulses at both ends, frame 1: zeros (every operand of every block zero)
    half: bool = False                  # model.half(): fp16 samples, parameters and output
    enc0v: int = 0                      # WUNET_TC_ENC0V
    pick: Optional[Tuple[int, ...]] = None


# fp32_tc. (4, 8, 3, 256): every block packed, a handful of CTAs. B = 256 / 257: the benchmarked persistent regime (62-249
# top-block tiles per CTA), checked on the frames of test_bf16_model_gpu.PICKS (packed-tile boundaries, the lone last frames).
# Odd lengths: T = 5 * 4096 (partial last tiles), a bottom level of one sample (T = 4096, n = 12), a 129-sample bottom level
# of partial packed tiles (T = 2064, n = 4). Channel plans 8 / 16 / 32. Wide plans: ci = 48 and 64, whose middle decoders run
# the SP = 2 chunk form, ci = 40 with enc0_wide_kernel at four channel slices, and one frame of 5 * 2^14 samples at ci = 64,
# whose blocks 8, 9, 15 and 16 are split over five column ranges. The half model runs the one-tile enc0_kernel
# and the last block's 16-bit I/O form; WUNET_TC_ENC0V=1 the one-tile block 0 with float I/O.
CASES = [
    Case("packed_n4", 4, 8, 3, 256, seed=11),
    Case("edges", 12, 24, 2, 16384, edges=True),
    Case("b256", 12, 24, 256, 16384, pick=tuple(PICKS[256])),
    Case("b257", 12, 24, 257, 16384, pick=tuple(PICKS[257])),
    Case("odd_20480", 12, 24, 3, 20480, seed=3),
    Case("bottom_L1", 12, 24, 5, 4096, seed=4),
    Case("bottom_L129", 4, 8, 5, 2064, seed=5),
    Case("plan_32", 5, 32, 3, 4096, seed=1),
    Case("plan_16", 5, 16, 2, 4096, seed=1),
    Case("plan_8", 6, 8, 3, 2048, seed=1),
    Case("wide_48", 12, 48, 2, 16384, seed=6),
    Case("wide_64", 12, 64, 2, 16384, seed=7),
    Case("wide_40", 10, 40, 3, 10240, seed=8),
    Case("wide_64_long", 12, 64, 1, 81920, seed=12),
    Case("half", 12, 24, 4, 16384, seed=9, half=True),
    Case("enc0v1", 6, 16, 3, 4096, seed=10, enc0v=1),
]
# fp32 (FFMA): conv_slide_kernel (L >= 256) and conv_gen_kernel (the rest), out_kernel
FP32_CASES = [
    Case("fp32_2", 12, 24, 2, 16384),
    Case("fp32_64", 12, 24, 64, 16384, pick=(0, 1, 2, 3, 31, 32, 62, 63)),
    Case("fp32_packed_n4", 4, 8, 3, 256, seed=11),
    Case("fp32_odd_20480", 12, 24, 3, 20480, seed=3),
    Case("fp32_wide_48", 12, 48, 2, 16384, seed=6),
]


def inputs(case):
    if not case.edges:
        return wo.make_input(case.B, case.T, seed=case.seed + 100)
    x = np.zeros((case.B, 1, case.T), np.float32)
    x[0, 0, 0], x[0, 0, -1] = 1.0, -1.0
    return x


def state(case):
    st = wo.make_state(case.n, case.ci, seed=case.seed)
    if case.half:                               # the values a half model holds, widened exactly
        st = {k: (np.asarray(v).astype(np.float16).astype(np.float32) if np.asarray(v).dtype.kind == "f" else v) for k, v in st.items()}
    return st


def check(case, mode, monkeypatch):
    """-> (per-block rows, output worst error / bar, the GPU output of the whole batch, the model, the input)"""
    for k in ENV_KNOBS:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")                # materialise the last block's activations too
    if case.enc0v:
        monkeypatch.setenv("WUNET_TC_ENC0V", str(case.enc0v))
    n, ci, B, T = case.n, case.ci, case.B, case.T
    assert case.pick is None or max(case.pick) < B, case
    st = state(case)
    x = inputs(case)
    m = Model(n, ci, precision=mode)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()})
    m = m.to(DEV).eval()
    xd = torch.from_numpy(x).to(DEV)
    if case.half:
        m = m.half()
        xd = xd.half()
    with torch.no_grad():
        y_all = m(xd)
    idx = None if case.pick is None else torch.tensor(case.pick, device=DEV)
    pick = lambda t: t if idx is None else t.index_select(0, idx)        # noqa: E731  (levels sliced on the device)
    got = [pick(m.read_level(i, B, T)) for i in range(2 * n + 1)]
    y = pick(y_all).double()
    model = sm.forward_split_model(st, pick(xd).float(), n, ci, mode, forced=got, device=DEV)
    rows = []
    for i in range(2 * n + 1):
        g = got[i].double()
        r = sm.ratio((g - model.levels[i]).abs(), sm.block_bar(g, model.levels[i], model.scale[i], model.shift[i], mode))
        rows.append((i, float(r.max()), float((g == model.levels[i]).double().mean())))
    C = got[2 * n].shape[1]
    ry = float(sm.ratio((y - model.y).abs(), sm.head_bar(model, C, mode, y16=case.half)).max())
    m._release()
    return rows, ry, y_all, st, x


def report(case, mode, rows, ry, dt):
    print(f"\n{mode} {case.name} (n={case.n} ci={case.ci} B={case.B} T={case.T}): worst error/bar per block, fraction equal")
    print("   " + "  ".join(f"{i}:{r:.2f}/{f:.4f}" for i, r, f in rows))
    print(f"   blocks worst {max(r for _, r, _ in rows):.3f}  output {ry:.3f}  ({dt:.1f} s)")


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_fp32_tc_blocks_match_the_split_model(case, monkeypatch):
    t0 = time.time()
    rows, ry, y_all, st, x = check(case, "fp32_tc", monkeypatch)
    report(case, "fp32_tc", rows, ry, time.time() - t0)
    bad = [(i, r) for i, r, _ in rows if not r <= 1.0]
    assert not bad, f"blocks over their bar (block, worst error/bar): {bad}"
    assert ry <= 1.0, f"output at {ry:.3g} of its bar"
    if case.B != 256:
        return
    # the benchmarked variant (the last block's activations not stored) computes the same output bits
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "0")
    m0 = Model(case.n, case.ci, precision="fp32_tc")
    m0.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()})
    m0 = m0.to(DEV).eval()
    with torch.no_grad():
        assert torch.equal(m0(torch.from_numpy(x).to(DEV)), y_all), "WUNET_TC_STORE_LAST=0 changes the output"
    m0._release()


@pytest.mark.parametrize("case", FP32_CASES, ids=[c.name for c in FP32_CASES])
def test_fp32_blocks_match_the_model(case, monkeypatch):
    t0 = time.time()
    rows, ry, _y, _st, _x = check(case, "fp32", monkeypatch)
    report(case, "fp32", rows, ry, time.time() - t0)
    bad = [(i, r) for i, r, _ in rows if not r <= 1.0]
    assert not bad, f"blocks over their bar (block, worst error/bar): {bad}"
    assert ry <= 1.0, f"output at {ry:.3g} of its bar"
