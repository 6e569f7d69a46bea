"""Model(train_precision="fp16_scaled") without a GPU: the constants and the constructor surface, the dz scaling rule on crafted
values (host-only query of the function the kernels use), the training workspace layout at the new precision, the per-pass
float64 restatement with fp16 rounding, and the fp16 training unit's ptxas report (compiled to a temporary directory; the
in-tree library is untouched)."""
import ctypes
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from wave_u_net_for_speech_enhancement_b200 import Model, _lib, build

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DWUNET_BUILD"]


def test_constants_and_mapping():
    assert _lib.PREC_FP16_SCALED == 5 and _lib.TRAIN_PRECISIONS["fp16_scaled"] == 5
    assert "fp16_scaled" not in _lib.PRECISIONS
    assert "fp16" not in _lib.TRAIN_PRECISIONS                   # plain fp16 (autocast semantics) stays refused
    with open(os.path.join(os.path.dirname(build.CSRC), "..", "include", "wunet_b200.h")) as f:
        assert re.search(r"#define WUNET_PREC_FP16_SCALED 5\b", f.read())


def test_model_accepts_it_with_the_native_backend_only():
    assert Model(4, 8, train_precision="fp16_scaled").train_precision == "fp16_scaled"
    for backend in ("torch", "none"):
        with pytest.raises(ValueError):
            Model(4, 8, train_backend=backend, train_precision="fp16_scaled")
    with pytest.raises(ValueError):
        Model(4, 8, train_precision="fp16")
    with pytest.raises(ValueError):
        Model(4, 8, precision="fp16_scaled")


def _k(amax):
    return _lib.load().wunet_debug_train_dz_scale(float(amax))


def _rule(amax):
    """amax 2^k in [2^13, 2^14), 0 for 0 / non-finite, |k| <= 126"""
    if not (amax > 0 and math.isfinite(amax)):
        return 0
    return max(-126, min(126, 13 - math.floor(math.log2(amax))))


CRAFTED = [0.0, 1.0, 2.0 ** 13, 2.0 ** 14, 2.0 ** 14 - 1, 1e-7, 3e-7, 6.1e-5, 65504.0, 1e-30,
           float(np.float32(2.0 ** -149)), float(np.float32(2.0 ** -126)), float(np.float32(1e-40)),
           float(np.finfo(np.float32).max), 1e30, float("inf"), float("nan")]


@pytest.mark.parametrize("amax", CRAFTED, ids=[repr(v) for v in CRAFTED])
def test_scale_rule(amax):
    k = _k(amax)
    assert k == _rule(amax)
    if 0 < amax < float("inf") and -126 < k < 126:
        assert 2.0 ** 13 <= amax * 2.0 ** k < 2.0 ** 14
    # 2^k and 2^-k are normal fp32 numbers
    assert np.float32(2.0 ** k) >= np.finfo(np.float32).tiny and np.float32(2.0 ** -k) >= np.finfo(np.float32).tiny


def test_scale_rule_edges():
    assert _k(0.0) == _k(float("inf")) == _k(float("nan")) == 0
    assert _k(float(np.float32(2.0 ** -149))) == 126                # tiny: clamped
    assert _k(float(np.finfo(np.float32).max)) == 13 - 127
    assert _k(1e-7) == 13 + 24                                       # 1e-7 = 1.68 x 2^-24
    assert _k(2.0 ** 13) == 0 and _k(2.0 ** 14) == -1


def test_scale_rule_on_random_values():
    g = np.random.default_rng(5)
    bits = g.integers(1, 0x7F800000, 20000, dtype=np.uint32)         # every positive finite fp32, subnormals included
    for v in bits.view(np.float32)[:2000]:
        assert _k(v) == _rule(float(v)), v


def _npad(c):
    b16 = -(-c // 16)
    ntiles = -(-b16 // 4)
    return -(-b16 // ntiles) * 16 * ntiles


def _floats(n):
    return -(-n // 64) * 64


def _packed_bf16_floats(cout, cin, k):
    return -(-(-(-cin // 64) * k * _npad(cout) * 64) // 2)


LAYOUT_CASES = [(12, 24, 120, 16384), (12, 24, 2, 4096), (4, 8, 3, 256)]


@pytest.mark.parametrize("case", LAYOUT_CASES)
def test_layout_is_the_bf16_layout_plus_the_scale_slots(case):
    n, ci, B, T = case
    fields = ("z", "act", "ga", "mean", "invstd", "s1", "s2", "Cin", "Cin0", "Cin1", "Cout", "L", "ksize", "mode",
              "grid_x", "grid_y", "grid_z", "items", "positions", "items_per_cta")
    fp32 = [_lib.debug_train_layout(n, ci, B, T, i, "fp32") for i in range(2 * n + 1)]
    bf16 = [_lib.debug_train_layout(n, ci, B, T, i, "bf16") for i in range(2 * n + 1)]
    f16 = [_lib.debug_train_layout(n, ci, B, T, i, "fp16_scaled") for i in range(2 * n + 1)]
    extra = sum(_floats(_packed_bf16_floats(d["Cout"], d["Cin"], d["ksize"])) +
                _floats(_packed_bf16_floats(d["Cin"], d["Cout"], d["ksize"])) for d in fp32[1:])
    assert bf16[0]["workspace_bytes"] == fp32[0]["workspace_bytes"] + 4 * extra
    assert f16[0]["workspace_bytes"] == bf16[0]["workspace_bytes"] + 4 * _floats(2 * n + 1)
    for i, (b, h) in enumerate(zip(bf16, f16)):
        assert {f: b[f] for f in fields} == {f: h[f] for f in fields}
        assert h["workspace_bytes"] == f16[0]["workspace_bytes"]
        assert h["wgrad_tc"] == (0 if i == 0 else 3) and b["wgrad_tc"] == (0 if i == 0 else 1)
    # field 22: the scale slots, one float per block after the packings; -1 for block 0 and for other precisions
    slot = []
    for i in range(2 * n + 1):
        for prec in ("fp32", "bf16", "tf32", "fp16_scaled"):
            buf = (ctypes.c_longlong * 23)()
            _lib.check(_lib.load().wunet_debug_train_layout(n, ci, B, T, _lib.TRAIN_PRECISIONS[prec], i, buf, 23))
            assert list(buf[:22]) == list(_lib.debug_train_layout(n, ci, B, T, i, prec).values())
            if prec != "fp16_scaled" or i == 0:
                assert buf[22] == -1, (prec, i)
            else:
                slot.append(buf[22])
    assert slot[0] == 4 * (bf16[0]["workspace_bytes"] // 4) + 4 and np.all(np.diff(slot) == 4)


def test_layout_query_keeps_22_fields_for_22_slots():
    buf = (ctypes.c_longlong * 22)()
    assert _lib.load().wunet_debug_train_layout(12, 24, 2, 4096, _lib.PREC_FP16_SCALED, 3, buf, 22) == 0


def test_inference_plan_query_refuses_it():
    buf = (ctypes.c_int * 32)()
    assert _lib.load().wunet_debug_plan_prec(12, 24, 2, 4096, 1, 132, buf, 32, _lib.PREC_FP16_SCALED) == -1


def test_fp16_rounding_of_the_restatement():
    """The float64 restatement of the GPU tests rounds with torch.half: round to nearest even, overflow to inf, NaN kept."""
    e = 2.0 ** -11                                              # half an fp16 ulp at 1
    v = np.array([1 + e, 1 + 3 * e, -(1 + e), 65504.0, 65519.0, 65520.0, 1e6, -1e6, 2.0 ** -25, 2.0 ** -24 * 1.5,
                  float("nan")], dtype=np.float32)
    h = torch.from_numpy(v).half().double().numpy()
    assert list(h[:4]) == [1.0, 1 + 4 * e, -1.0, 65504.0]        # ties to even (down, up), sign, largest finite
    assert h[4] == 65504.0 and h[5] == np.inf and h[6] == np.inf and h[7] == -np.inf
    assert h[8] == 0.0 and h[9] == 2.0 ** -23                     # subnormal ties to even
    assert np.isnan(h[10])


def test_scaled_pass_restatement_is_exact_scaling():
    """sum fp16(dz 2^k) fp16(x) 2^-k: in float64 the restatement of a weight-gradient pass for dz and dz 2^m differs by
    exactly 2^m, and without the scaling dz of about 1e-7 would lose most of its bits in fp16."""
    g = np.random.default_rng(7)
    x = g.standard_normal((2, 5, 64)).astype(np.float32)
    dz = (1e-7 * g.standard_normal((2, 3, 64))).astype(np.float32)

    def wgrad(d):
        s = 2.0 ** _k(np.abs(d).max())
        dr = torch.from_numpy(d * np.float32(s)).half().double()
        xr = torch.from_numpy(x).half().double()
        return torch.nn.grad.conv1d_weight(xr, (3, 5, 15), dr, padding=7).numpy() / s

    base = wgrad(dz)
    for m in (-24, 16):
        assert np.array_equal(wgrad((dz * np.float32(2.0 ** m)).astype(np.float32)), base * 2.0 ** m)
    unscaled = torch.from_numpy(dz).half().double().numpy()
    assert np.abs(unscaled - dz).max() > 0.05 * np.abs(dz).max()     # fp16 without scaling: subnormal, few bits left


def _nvcc():
    try:
        return build.nvcc_path()
    except RuntimeError:
        return None


@pytest.mark.skipif(_nvcc() is None, reason="needs nvcc")
def test_fp16_unit_ptxas_report(tmp_path):
    """wunet_train_tc_f16.cu compiles to the 23 fp16 kernels (conv, weight gradient, pack), without spills or wgmma
    serialisation."""
    r = subprocess.run([_nvcc()] + NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "wunet_train_tc_f16.cu"),
                        "-o", str(tmp_path / "f16.o")], capture_output=True, text=True)
    log = r.stdout + r.stderr
    assert r.returncode == 0, log[-4000:]
    entries = re.findall(r"Compiling entry function '(\w+)'", log)
    assert len(entries) == 23 and all("F16" in e for e in entries), entries
    assert "C7519" not in log and "C7520" not in log
    assert all(int(s) == 0 for s in re.findall(r"(\d+) bytes spill stores", log))
    assert "20281" not in log
