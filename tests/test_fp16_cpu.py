"""Model(precision="fp16") without a GPU: the constructor surface, the plan and training-layout queries (host-only), the fp16
translation unit compiled for sm_90a with ptxas in verbose mode, and the fp16 arithmetic model (tests/fp16_model.py) against the
C oracle. Compilations go to a temporary directory; the in-tree library is untouched."""
import copy
import ctypes
import json
import os
import pickle
import re
import subprocess

import numpy as np
import pytest

import fp16_model as fm
from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model, _lib, build

HERE = os.path.dirname(os.path.abspath(__file__))
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DWUNET_BUILD"]

# every shape tests/test_fp16_gpu.py runs (n, ci, B, T), and the SM counts it plans for
GPU_SHAPES = [(4, 8, 3, 256), (12, 24, 2, 16384), (6, 8, 64, 512), (12, 24, 256, 16384), (12, 24, 257, 16384), (4, 8, 2, 4096),
              (12, 24, 64, 16384), (4, 8, 3, 256)]
SMS = [132, 114]


def _nvcc():
    try:
        return build.nvcc_path()
    except RuntimeError:
        return None


def test_fp16_is_an_inference_precision():
    m = Model(4, 8, precision="fp16")
    assert m.precision == "fp16" and m.train_precision == "fp32"
    assert _lib.PRECISIONS["fp16"] == _lib.PREC_FP16 == 4
    assert "fp16" not in _lib.TRAIN_PRECISIONS


def test_fp16_is_not_a_training_precision():
    with pytest.raises(ValueError):
        Model(4, 8, train_precision="fp16")


def test_state_dict_keys_unchanged():
    with open(os.path.join(HERE, "golden", "state_dict_surface.json")) as f:
        surface = json.load(f)
    sd = Model(precision="fp16").state_dict()
    assert len(sd) == 177
    assert [[k, list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd.items()] == surface["state_dict"]


def test_copies_keep_the_setting():
    m = Model(4, 8, precision="fp16")
    assert copy.deepcopy(m).precision == "fp16"
    assert pickle.loads(pickle.dumps(m)).precision == "fp16"


@pytest.mark.parametrize("shape", sorted(set(GPU_SHAPES)))
@pytest.mark.parametrize("sms", SMS)
def test_fp16_plan_is_the_bf16_plan(shape, sms):
    n, ci, B, T = shape
    for block in range(1, 2 * n + 1):
        assert _lib.debug_plan(n, ci, B, T, block, sms, "fp16") == _lib.debug_plan(n, ci, B, T, block, sms, "bf16"), block


def test_fp16_plan_without_the_dense_gemm(monkeypatch):
    monkeypatch.setenv("WUNET_TC_GEMM", "0")
    for block in range(1, 25):
        assert _lib.debug_plan(12, 24, 256, 16384, block, 132, "fp16") == _lib.debug_plan(12, 24, 256, 16384, block, 132, "bf16")


def test_fp16_has_no_tensor_core_block_0(monkeypatch):
    monkeypatch.setenv("WUNET_TC_ENC0", "1")
    _lib.debug_plan(12, 24, 2, 16384, 0, 132, "bf16")            # the opt-in group-of-8 form exists for bf16 ...
    with pytest.raises(_lib.WunetError):                           # ... and not for fp16
        _lib.debug_plan(12, 24, 2, 16384, 0, 132, "fp16")


def test_training_queries_refuse_fp16():
    buf = (ctypes.c_longlong * 32)()
    assert _lib.load().wunet_debug_train_layout(12, 24, 2, 4096, _lib.PREC_FP16, 0, buf, 32) == -1      # WUNET_EINVAL
    with pytest.raises(_lib.WunetError):
        _lib.debug_train_layout(12, 24, 2, 4096, 0, "fp16")


def _ptxas_table(log):
    """mangled kernel name -> (registers, static shared memory bytes, spill store bytes), from ptxas -v"""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            out[cur] = [0, 0, 0]
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes spill stores", line)
        if m:
            out[cur][2] = int(m.group(1))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            smem = re.search(r"(\d+) bytes smem", line)            # static shared memory; absent when there is none
            out[cur][0], out[cur][1] = int(m.group(1)), int(smem.group(1)) if smem else 0
    return {k: tuple(v) for k, v in out.items()}


def _by_name(table, prefix):
    """(kernel name + template arguments) -> figures, for the kernels of one namespace; the parameter list is dropped (its
    mangled substitutions differ between the namespaces)"""
    out = {}
    for k, v in table.items():
        m = re.match(re.escape(prefix) + r"(\d+)", k)
        if m and not k[len(prefix):].startswith("3f16"):
            name_len = int(m.group(1))
            start = len(prefix) + len(m.group(1))
            rest = k[start + name_len:]
            targs = rest[:rest.index("Ev")] if rest.startswith("I") else ""
            out[k[start:start + name_len] + targs] = v
    return out


@pytest.mark.skipif(_nvcc() is None, reason="needs nvcc")
def test_fp16_kernels_compile_like_their_bf16_twins(tmp_path):
    """No wgmma serialisation warnings, and every fp16 kernel uses the registers, shared memory and spill stores of its bf16
    twin: the fp16 kernels add no spills (the small decoder forms and enc0 spill a few bytes in both element types)."""
    logs = {}
    for src in ("wunet_tc_f16.cu", "wunet_tc.cu"):
        cmd = [_nvcc()] + NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, src), "-o", str(tmp_path / (src + ".o"))]
        r = subprocess.run(cmd, capture_output=True, text=True)
        logs[src] = r.stdout + r.stderr
        assert r.returncode == 0, logs[src][-4000:]
    f16 = logs["wunet_tc_f16.cu"]
    bad = [line for line in f16.splitlines() if re.search(r"C75(19|20)", line)]
    assert not bad, "\n".join(bad[:10])
    t16 = _by_name(_ptxas_table(f16), "_ZN5wunet3f16")
    tbf = _by_name(_ptxas_table(logs["wunet_tc.cu"]), "_ZN5wunet")
    # the eight conv forms the bf16 plan launches (encoder, decoder, decoder with merged tail, row-pair encoder; large and small)
    # and the other kernels of the fp16 path
    assert sum(k.startswith("conv_tc_kernel") for k in t16) == 8, sorted(t16)
    for name in ("gemm_tc_kernel", "enc0_kernel", "enc0_kernel_v2", "pack_tc_kernel", "pack_tc_merged_kernel",
                 "expand_gemm_weights_kernel", "nlc_f16_to_ncl_f32_kernel"):
        assert name in t16, name
    tbf["nlc_f16_to_ncl_f32_kernel"] = tbf["nlc_bf16_to_ncl_f32_kernel"]
    for k, v in t16.items():
        assert k in tbf, k
        if k.startswith("conv_tc_kernel"):
            assert v == tbf[k], (k, v, tbf[k])
        else:
            assert v[2] <= tbf[k][2], (k, v, tbf[k])


def test_fp16_rounding_saturates_and_keeps_subnormals():
    import torch
    v = torch.tensor([70000.0, -1e30, 65519.0, 65520.0, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -25, 1 + 2.0 ** -11, float("nan")],
                     dtype=torch.float64)
    got = fm.f16(v).numpy()
    assert list(got[:4]) == [65504.0, -65504.0, 65504.0, 65504.0]
    assert got[4] == 2.0 ** -24 and got[5] == 0.0 and got[6] == 2.0 ** -23     # ties to even in the subnormal range
    assert got[7] == 1.0 and np.isnan(got[8])
    # a float64 value just above a tie rounds up; through fp32 first it would become the tie and round to even (down)
    w = torch.tensor([1 + 2.0 ** -11 + 2.0 ** -40], dtype=torch.float64)
    assert fm.f16(w).item() == 1 + 2.0 ** -10


def test_fp16_model_matches_the_c_oracle_on_the_small_config():
    n, ci, B, T = 4, 8, 3, 256
    st = wo.make_state(n, ci, seed=11)
    x = wo.make_input(B, T, seed=111)
    want_y, want = wo.COracle(n, ci).forward(st, x, return_levels=True)
    y, lv = fm.forward_fp16_model(st, x, n, ci, return_levels=True)
    errs = [float(np.abs(a - b).max()) for a, b in zip(lv, want)]
    assert float(np.abs(y - want_y).max()) <= 3e-4
    assert max(errs) <= 3e-4 * max(1.0, max(float(np.abs(w).max()) for w in want)), errs
