"""Tiling invariance of the tensor-core forward: every plan with the same arithmetic must give the same bits.

The K loop of a block runs in an order fixed by its channel plan (taps, then 64-channel chunks), never by its tiling: how many
SMs the persistent grid covers, how the columns are split, how many frames a packed tile holds, how deep the rings are, whether
the weights stay resident. So a run under another plan must reproduce every block output (``WUNET_TC_STORE_LAST=1``: all 2n + 1
of them) and the network output bit for bit. The run without overrides is the reference; test_bf16_model_gpu.py ties that run
to the arithmetic model.

Plans are switched with two test hooks, read at every forward: ``WUNET_TC_SMS=<n>`` (plan and size the grids as on a device
with n SMs) and ``WUNET_TC_OVR`` (one block's tiling). ``packed=1`` is left out on purpose: it sends the decoder producers down
the fp32 interpolation path, a different arithmetic. tests/test_tiling_coverage_cpu.py checks on the CPU that these tables
reach every tiling feature the planner has."""
import contextlib
import os

import numpy as np
import pytest
import torch

from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model, _lib

pytestmark = [pytest.mark.gpu]

PRECISIONS = ("bf16", "fp32_tc")
SMS_COUNTS = (1, 7, 16, 60, 114)
# (n_layers, channels_interval, B, T, WUNET_TC_SMS), each in both precisions:
# - (12, 24, 64, 4096): the bottom blocks on the dense GEMM, column tiles Nh 16 ... 128 across the SM counts;
# - (12, 24, 5, 16384): packed tiles of 3, 4 and 5 frames, 4 or 6 column splits; at 114 SMs only the grids shrink;
# - (4, 8, 3, 256) never launches more than 6 CTAs: only one SM changes its plan;
# - (10, 24, 64, 4096) at 16 SMs: GEMM Nh = 80 (block 10); (8, 16, 1000, 256) at 7 SMs: Nh = 112 (blocks 6 and 10) and
#   a partial last row tile of the GEMM.
SMS_CASES = ([(12, 24, 64, 4096, s) for s in SMS_COUNTS] + [(12, 24, 5, 16384, s) for s in SMS_COUNTS] +
             [(4, 8, 3, 256, 1), (10, 24, 64, 4096, 16), (8, 16, 1000, 256, 7)])

# per-block WUNET_TC_OVR overrides, one block at a time, at this shape (bf16)
OVR_SHAPE = (12, 24, 5, 16384)
OVR_KEYS = ("small=1", "res=0", "tg=1", "tg=4", "nb=2", "na=2", "na=3", "ns+1")

# forward_host against the device path: (n, ci, B, T, precision, WUNET_TC_SMS or None). B = 32 and 256 run the last block in
# four tile ranges (one per host chunk).
HOST_CASES = [(12, 24, B, 16384, p, None) for B in (32, 256) for p in PRECISIONS] + [(12, 24, 256, 16384, "bf16", 7)]

# knobs that select a plan or an arithmetic; every test sets the ones it needs and clears the rest
PLAN_KNOBS = ("WUNET_TC_SMS", "WUNET_TC_OVR", "WUNET_TC_GEMM", "WUNET_TC_STORE_LAST", "WUNET_TC_PAIR", "WUNET_TC_ENC0",
              "WUNET_TC_ENC0V", "WUNET_TC_MERGE")


@contextlib.contextmanager
def _env(**kv):
    """Set environment variables for the duration of a host-only plan query (collection time: no monkeypatch yet)."""
    old = {k: os.environ.get(k) for k in kv}
    try:
        for k, v in kv.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def block_plans(n, ci, B, T, sms, precision="bf16", ovr=None, gemm=True):
    """debug_plan of blocks 1 .. 2n under the given override string."""
    with _env(WUNET_TC_OVR=ovr, WUNET_TC_GEMM=None if gemm else "0", WUNET_TC_PAIR=None, WUNET_TC_MERGE=None):
        return [_lib.debug_plan(n, ci, B, T, i, sms, precision) for i in range(1, 2 * n + 1)]


def override_cases(sms=132):
    """(block, override string) for every key of OVR_KEYS that the planner accepts on that block and that changes its plan
    (built on the CPU from debug_plan; "ns+1" = one column split more than the default, "res=0" only on resident blocks)."""
    n, ci, B, T = OVR_SHAPE
    base = block_plans(n, ci, B, T, sms)
    out = []
    for blk in range(1, 2 * n + 1):
        d0 = base[blk - 1]
        for key in OVR_KEYS:
            if key == "res=0" and not d0["resident"]:
                continue
            kv = "ns=%d" % (d0["nsplit"] + 1) if key == "ns+1" else key
            s = "%d:%s" % (blk, kv)
            try:
                d = block_plans(n, ci, B, T, sms, ovr=s)[blk - 1]
            except _lib.WunetError:
                continue
            if d != d0:
                out.append((blk, s))
    return out


OVR_CASES = override_cases()


# ---- running ---------------------------------------------------------------------------------------------------------------
def clear_knobs(monkeypatch):
    for k in PLAN_KNOBS:
        monkeypatch.delenv(k, raising=False)


def make_model(n, ci, precision, seed=0):
    m = Model(n, ci, precision=precision)
    st = wo.make_state(n, ci, seed=seed)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
    return m.to("cuda:0").eval()


def run_levels(n, ci, B, T, precision, levels=True):
    """Fresh model (the library reads WUNET_TC_STORE_LAST / WUNET_TC_GEMM when it creates the model's state), one seeded
    forward: output and, with levels, all 2n + 1 block outputs, on the device."""
    m = make_model(n, ci, precision)
    x = torch.from_numpy(wo.make_input(B, T, seed=1000 + B + T)).to("cuda:0")
    with torch.no_grad():
        y = m(x)
    lv = [m.read_level(i, B, T) for i in range(2 * n + 1)] if levels else []
    torch.cuda.synchronize()
    m._release()
    return y, lv


def assert_same_bits(ref, got, what):
    (y0, l0), (y1, l1) = ref, got
    bad = [i for i, (a, b) in enumerate(zip(l0, l1)) if not torch.equal(a, b)]
    assert not bad, f"{what}: blocks {bad} differ from the reference plan"
    assert torch.equal(y0, y1), f"{what}: output differs from the reference plan"


_REFS = {}


@pytest.fixture(scope="module")
def reference():
    """Reference runs (no overrides, all blocks stored), computed once per (shape, precision, GEMM on / off)."""
    def get(n, ci, B, T, precision, gemm=True):
        key = (n, ci, B, T, precision, gemm)
        if key not in _REFS:
            with pytest.MonkeyPatch.context() as mp:
                clear_knobs(mp)
                mp.setenv("WUNET_TC_STORE_LAST", "1")
                if not gemm:
                    mp.setenv("WUNET_TC_GEMM", "0")
                _REFS[key] = run_levels(n, ci, B, T, precision)
        return _REFS[key]
    yield get
    _REFS.clear()


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("n,ci,B,T,sms", SMS_CASES)
def test_sm_count_does_not_change_the_bits(n, ci, B, T, sms, precision, reference, monkeypatch):
    dev_sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert block_plans(n, ci, B, T, sms, precision) != block_plans(n, ci, B, T, dev_sms, precision), \
        "the case would run the device's own plan"
    ref = reference(n, ci, B, T, precision)
    clear_knobs(monkeypatch)
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")
    monkeypatch.setenv("WUNET_TC_SMS", str(sms))
    assert_same_bits(ref, run_levels(n, ci, B, T, precision), f"WUNET_TC_SMS={sms}")


@pytest.mark.parametrize("block,ovr", OVR_CASES)
def test_block_override_does_not_change_the_bits(block, ovr, reference, monkeypatch):
    n, ci, B, T = OVR_SHAPE
    # an override takes its block off the dense GEMM: compare such a block with the reference that has the GEMM off too
    on_gemm = block_plans(n, ci, B, T, torch.cuda.get_device_properties(0).multi_processor_count)[block - 1]["small"] == 2
    ref = reference(n, ci, B, T, "bf16", gemm=not on_gemm)
    clear_knobs(monkeypatch)
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")
    if on_gemm:
        monkeypatch.setenv("WUNET_TC_GEMM", "0")
    monkeypatch.setenv("WUNET_TC_OVR", ovr)
    assert_same_bits(ref, run_levels(n, ci, B, T, "bf16"), f"WUNET_TC_OVR={ovr}")


@pytest.mark.parametrize("n,ci,B,T,precision,sms", HOST_CASES)
def test_forward_host_matches_the_device_path(n, ci, B, T, precision, sms, monkeypatch):
    """Host in, host out (the last block per host chunk of B / 4 frames) against the device path without overrides."""
    clear_knobs(monkeypatch)
    m = make_model(n, ci, precision)
    x = wo.make_input(B, T, seed=77 + B)
    with torch.no_grad():
        y = m(torch.from_numpy(x).to("cuda:0")).cpu()
    if sms is not None:
        monkeypatch.setenv("WUNET_TC_SMS", str(sms))
    yh = m.forward_host(torch.from_numpy(x).pin_memory())
    m._release()
    assert torch.equal(yh, y)
