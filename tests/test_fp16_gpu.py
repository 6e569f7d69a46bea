"""Model(precision="fp16") on an H100: the fp16 kernels against their arithmetic model (tests/fp16_model.py) level by level,
against the fp32 oracle and the goldens, the same bits from every planner switch and host entry point, saturation, and the
C ABI. The bars against the model are derived: a value may differ from the model where the fp32 accumulation order flips an
fp16 rounding (one ulp, two where a flip meets the next tie), or, where the pre-activation cancels, by an fp32 rounding error of
the sum: 2^-14 of the level's largest magnitude (2^-11 of it is bf16's floor, test_bf16_model_gpu.py; fp16 has 3 more bits)."""
import ctypes
import os

import numpy as np
import pytest
import torch

import fp16_model as fm
from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model, _lib
from wave_u_net_for_speech_enhancement_b200.enhance import enhance_waveforms, frame_clips, unframe_clips

pytestmark = [pytest.mark.gpu]

HERE = os.path.dirname(os.path.abspath(__file__))
ABS_FLOOR = 2.0 ** -14
PICK = [0, 1, 2, 3, 127, 128, 254, 255]
PICKS = {256: PICK, 257: PICK + [256]}
# the cases of test_bf16_model_gpu.py::MODEL_CASES
MODEL_CASES = [(4, 8, 3, 256, 11), (12, 24, 2, 16384, 0), (6, 8, 64, 512, 5), (12, 24, 256, 16384, 0), (12, 24, 257, 16384, 0)]
OTHER_SMS = 114
SWITCHES = ("WUNET_TC_SMS", "WUNET_TC_OVR", "WUNET_TC_GEMM", "WUNET_TC_STORE_LAST", "WUNET_TC_ENC0")


def make_model(n, ci, st, precision="fp16"):
    m = Model(n, ci, precision=precision)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()})
    return m.to("cuda:0").eval()


def run(m, x, pick=None):
    B, _, T = x.shape
    idx = None if pick is None else torch.tensor(pick, device="cuda:0")
    with torch.no_grad():
        y = m(torch.from_numpy(x).cuda())
    levels = []
    for i in range(2 * m.n_layers + 1):
        lv = m.read_level(i, B, T)
        levels.append(lv if idx is None else lv.index_select(0, idx))
    return y, levels


def compare_with_model(st, x, got_levels, y, n, ci, dense_bottom):
    want_y, want = fm.forward_fp16_model(st, x, n, ci, return_levels=True, forced=got_levels[:2 * n], dense_bottom=dense_bottom)
    report = []
    for i in range(2 * n + 1):
        got = got_levels[i]
        ref = want[i] if i < 2 * n else fm.f16(torch.from_numpy(want[i])).numpy()     # the stored copy of the last block
        diff = np.abs(got - ref)
        bound = np.maximum(2.0 * fm.ulp_f16(ref), ABS_FLOOR * np.abs(ref).max())
        report.append((i, round(float((diff == 0).mean()), 5), float(diff.max()), float((diff - bound).max())))
    yerr = float(np.abs(y - want_y).max())
    print("fp16 model (teacher-forced) vs kernels: (block, fraction bit-equal, max abs diff, excess over bound)")
    for r in report:
        print("   ", r)
    print("    output max-abs diff", yerr)
    assert all(r[1] >= 0.98 for r in report), report
    assert all(r[3] <= 0.0 for r in report), report
    assert yerr <= 2e-5, (yerr, report)


@pytest.mark.parametrize("n,ci,B,T,seed", MODEL_CASES)
def test_levels_match_the_arithmetic_model(n, ci, B, T, seed, monkeypatch):
    pick = PICKS.get(B)
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")
    st = wo.make_state(n, ci, seed=seed)
    x = wo.make_input(B, T, seed=seed + 100)
    m = make_model(n, ci, st)
    y_dev, lv_dev = run(m, x, pick)
    xs = x if pick is None else x[pick]
    y = (y_dev if pick is None else y_dev[pick]).cpu().numpy()
    compare_with_model(st, xs, [lv.cpu().numpy() for lv in lv_dev], y, n, ci, B >= 64)
    if B != 256:
        return
    # the same bits over the whole batch: without the last block stored, planned for another SM count, host entry points
    y_all, lv_all = run(m, x)
    m._release()
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "0")
    m0 = make_model(n, ci, st)
    with torch.no_grad():
        assert torch.equal(m0(torch.from_numpy(x).cuda()), y_all), "WUNET_TC_STORE_LAST=0 changes the output"
    xh = torch.from_numpy(x).pin_memory()
    assert torch.equal(m0.forward_host(xh), y_all.cpu()), "forward_host differs from the device path"
    outs = list(m0.forward_host_stream([xh[:128].contiguous(), xh[128:].contiguous()]))
    m0._release()
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")
    monkeypatch.setenv("WUNET_TC_SMS", str(OTHER_SMS))
    y2, lv2 = run(make_model(n, ci, st), x)
    assert [i for i in range(2 * n + 1) if not torch.equal(lv2[i], lv_all[i])] == [], f"WUNET_TC_SMS={OTHER_SMS}: blocks differ"
    assert torch.equal(y2, y_all), f"WUNET_TC_SMS={OTHER_SMS}: output differs"
    # forward_host_stream ran batches of 128 frames: compare with the device path at that batch
    monkeypatch.delenv("WUNET_TC_SMS")
    m1 = make_model(n, ci, st)
    with torch.no_grad():
        for half, o in zip((x[:128], x[128:]), outs):
            assert torch.equal(m1(torch.from_numpy(half).cuda()).cpu(), o), "forward_host_stream differs from the device path"


def test_dense_gemm_off_matches_the_model(monkeypatch):
    n, ci, B, T, seed = 6, 8, 64, 512, 5
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")
    monkeypatch.setenv("WUNET_TC_GEMM", "0")
    st = wo.make_state(n, ci, seed=seed)
    x = wo.make_input(B, T, seed=seed + 100)
    y, lv = run(make_model(n, ci, st), x)
    compare_with_model(st, x, [t.cpu().numpy() for t in lv], y.cpu().numpy(), n, ci, dense_bottom=False)


def test_enhance_waveforms_equals_the_device_path(monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    n, ci, T = 12, 24, 16384
    st = wo.make_state(n, ci, seed=3)
    m = make_model(n, ci, st)
    rng = np.random.default_rng(7)
    clips = [(0.1 * rng.standard_normal(L)).astype(np.float32) for L in (4 * T, 3 * T + 1000)]
    got = enhance_waveforms(m, clips, sample_length=T, batch_frames=4)
    frames, index = frame_clips(clips, T, round_to=4)
    with torch.no_grad():
        y = torch.cat([m(frames[i:i + 4].cuda()).cpu() for i in range(0, frames.shape[0], 4)])
    want = unframe_clips(y, index, True)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))


def test_against_the_fp32_oracle_at_every_level(monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")
    n, ci, B, T = 4, 8, 3, 256
    st = wo.make_state(n, ci, seed=11)
    x = wo.make_input(B, T, seed=111)
    y, lv = run(make_model(n, ci, st), x)
    want_y, want = wo.COracle(n, ci).forward(st, x, return_levels=True)
    errs = [float(np.abs(g.cpu().numpy() - w).max()) for g, w in zip(lv, want)]
    print("fp16 small config per-level max-abs vs fp32 oracle", " ".join("%.1e" % e for e in errs))
    assert max(errs) <= 3e-4 * max(1.0, max(float(np.abs(w).max()) for w in want)), errs
    assert float(np.abs(y.cpu().numpy() - want_y).max()) <= 3e-4


def _outputs(st, x, precisions=("fp16", "bf16")):
    out = {}
    for prec in precisions:
        m = make_model(12, 24, st, prec)
        with torch.no_grad():
            out[prec] = m(torch.from_numpy(np.ascontiguousarray(x)).cuda()).cpu().numpy()
        m._release()
    return out


def test_full_config_against_the_golden(golden_dir, monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    g = np.load(os.path.join(golden_dir, "full_n12_c24_b2.npz"))
    st = wo.make_state(12, 24, seed=int(g["state_seed"]))
    x = wo.make_input(2, 16384, seed=int(g["input_seed"]))
    y = _outputs(st, x)
    errs = {p: float(np.abs(v - g["y"]).max()) for p, v in y.items()}
    print("full config B=2 max-abs vs golden", errs)
    assert errs["fp16"] <= 3e-4 and errs["fp16"] <= 0.25 * errs["bf16"], errs


def test_config2_batch64_with_the_edge_vectors(golden_dir, monkeypatch):
    """B = 64 (the dense GEMM at the bottom of the U): 60 random frames and 4 edge vectors; the random frames checked against
    the fp32 oracle at four picks, the edge vectors against their goldens."""
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    g = np.load(os.path.join(golden_dir, "edges_n12_c24.npz"))
    st = wo.make_state(12, 24, seed=int(g["state_seed"]))
    edges = wo.edge_inputs(16384)
    names = [k for k in ("impulse_first", "dc_pos", "dc_neg", "alternating") if k in edges]
    x = np.concatenate([wo.make_input(64 - len(names), 16384, seed=4321)] + [edges[k] for k in names]).astype(np.float32)
    y = _outputs(st, x)
    pick = [0, 17, 42, 59]
    want = wo.COracle(12, 24).forward(st, x[pick])
    errs = {p: max(float(np.abs(v[pick] - want).max()),
                   max(float(np.abs(v[64 - len(names) + j] - g[k][0]).max()) for j, k in enumerate(names))) for p, v in y.items()}
    print("config 2 B=64 max-abs vs oracle / edge goldens", errs)
    assert errs["fp16"] <= 3e-4 and errs["fp16"] <= 0.25 * errs["bf16"], errs


def test_saturation_is_exact(monkeypatch):
    """Two channels driven past +-65504 in both signs (block 0 on the CUDA cores, block 1 on the tensor cores): the stored
    levels hold exactly +-65504 there, the output stays finite and matches the saturating model."""
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("WUNET_TC_STORE_LAST", "1")
    n, ci, B, T = 4, 8, 3, 256
    st = {k: np.array(v, copy=True) for k, v in wo.make_state(n, ci, seed=11).items()}
    plan = wo.channel_plan(n, ci)
    st[f"{plan[0][0]}.1.weight"][2] *= np.float32(3e6)
    st[f"{plan[1][0]}.1.weight"][3] *= np.float32(1e7)
    x = wo.make_input(B, T, seed=111)
    y, lv = run(make_model(n, ci, st), x)
    got = [t.cpu().numpy() for t in lv]
    for blk, ch in ((0, 2), (1, 3)):
        c = got[blk][:, ch]
        assert (c == 65504.0).any() and (c == -65504.0).any(), (blk, c.max(), c.min())
        assert np.abs(c).max() == 65504.0
    yn = y.cpu().numpy()
    assert np.isfinite(yn).all() and all(np.isfinite(g).all() for g in got)
    compare_with_model(st, x, got, yn, n, ci, dense_bottom=False)


def test_c_abi_fp16_is_inference_only():
    lib = _lib.load()
    m = Model(4, 8, precision="fp16")
    c = m._context(torch.device("cuda:0"))
    try:
        EINVAL = -1
        for B, T in ((2, 256), (256, 16384), (257, 16384)):
            assert lib.wunet_workspace_bytes(c, B, T, _lib.PREC_FP16) == lib.wunet_workspace_bytes(c, B, T, _lib.PREC_BF16) > 0
        B, T = 2, 256
        assert lib.wunet_train_workspace_bytes_prec(c, B, T, _lib.PREC_FP16) == 0
        assert lib.wunet_train_workspace_bytes_ex(c, B, T, _lib.PREC_FP16, 0) == 0
        m = m.cuda().eval()
        x = torch.zeros(B, 1, T, device="cuda")
        with torch.no_grad():
            m(x)
        ws = torch.empty(1 << 26, dtype=torch.uint8, device="cuda")
        null = ctypes.c_void_p(0)
        nb = 2 * 4 + 1
        ptrs = (ctypes.c_void_p * nb)()
        y = torch.empty_like(x)
        rc = lib.wunet_train_forward_prec(c, x.data_ptr(), y.data_ptr(), B, T, ptrs, ptrs, ptrs, ptrs, ptrs, ptrs, null, null,
                                          ctypes.c_float(0.1), ws.data_ptr(), ws.numel(), null, _lib.PREC_FP16)
        assert rc == EINVAL
        assert "WUNET_PREC_FP16" in lib.wunet_last_error().decode()
        rc = lib.wunet_train_backward_part_prec(c, x.data_ptr(), y.data_ptr(), x.data_ptr(), B, T, ptrs, ptrs, ptrs, null, ptrs, ptrs,
                                                ptrs, ptrs, null, null, ws.data_ptr(), ws.numel(), null, -1, _lib.PREC_FP16)
        assert rc == EINVAL
        torch.cuda.synchronize()
    finally:
        m._release()


def test_fp16_weights_follow_weight_updates(monkeypatch):
    """The fp16 packing is made lazily and redone after new weights: bf16 -> fp16 -> new weights -> fp16 equals a fresh model."""
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    n, ci, B, T = 4, 8, 3, 256
    st0, st1 = wo.make_state(n, ci, seed=11), wo.make_state(n, ci, seed=12)
    x = torch.from_numpy(wo.make_input(B, T, seed=111)).cuda()
    m = make_model(n, ci, st0, "bf16")
    with torch.no_grad():
        m(x)
        m.precision = "fp16"
        m(x)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st1.items()})
        y = m(x)
        assert torch.equal(y, make_model(n, ci, st1)(x))
