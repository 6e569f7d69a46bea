"""Model(train_precision="tf32") without a GPU: the SASS of the forward library's tensor-core object unchanged by the wgmma
header it shares with the training kernels, the constructor surface, and the training workspace layout at the new precision
(host-only query). The tf32 training kernels themselves (wunet_train_tc.cu) are compiled and checked by
test_train_tc_unit_cpu.py. Compilations go to a temporary directory; the in-tree library is untouched."""
import copy
import ctypes
import hashlib
import json
import os
import pickle
import re
import subprocess

import pytest

from wave_u_net_for_speech_enhancement_b200 import Model, _lib, build

HERE = os.path.dirname(os.path.abspath(__file__))
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DWUNET_BUILD"]


def _nvcc():
    try:
        return build.nvcc_path()
    except RuntimeError:
        return None


def _nvcc_release():
    nv = _nvcc()
    if nv is None:
        return None
    m = re.search(r"release (\d+\.\d+), V([\d.]+)", subprocess.run([nv, "--version"], capture_output=True, text=True).stdout)
    return m and m.group(2)


# sha256 of `cuobjdump -sass` of the object as built before the tf32 helpers joined wunet_wgmma.cuh (nvcc 12.9.86, the flags
# above), with the per-file hash of the anonymous namespace's mangled name (it depends on the source path) blanked out. The
# training kernels' SASS is checked kernel by kernel in test_train_tc_unit_cpu.py.
SASS_DIGESTS = {"wunet_tc.cu": "b3d936616e93378da6a85a111a6b5027f3c975d553483856000b716810779a48"}
SASS_NVCC = "12.9.86"


@pytest.mark.skipif(_nvcc_release() != SASS_NVCC, reason=f"the recorded SASS digests are those of nvcc {SASS_NVCC}")
@pytest.mark.parametrize("src", sorted(SASS_DIGESTS))
def test_wgmma_header_leaves_the_other_tensor_core_objects_unchanged(tmp_path, src):
    obj = str(tmp_path / src.replace(".cu", ".o"))
    r = subprocess.run([_nvcc()] + NVCC_FLAGS + ["-c", os.path.join(build.CSRC, src), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
    sass = subprocess.run([os.path.join(os.path.dirname(_nvcc()), "cuobjdump"), "-sass", obj], capture_output=True, text=True,
                          check=True).stdout
    sass = re.sub(r"_GLOBAL__N__[0-9a-f]+_", "_GLOBAL__N__", sass)
    assert hashlib.sha256(sass.encode()).hexdigest() == SASS_DIGESTS[src]


def test_tf32_is_a_training_precision():
    assert Model(4, 8, train_precision="tf32").train_precision == "tf32"
    assert Model(4, 8).train_precision == "fp32"                 # the default step is unchanged
    assert "tf32" not in _lib.PRECISIONS and _lib.TRAIN_PRECISIONS["tf32"] == _lib.PREC_TF32 == 3


def test_tf32_is_not_an_inference_precision():
    with pytest.raises(ValueError):
        Model(4, 8, precision="tf32")


@pytest.mark.parametrize("backend", ["torch", "none"])
def test_tf32_needs_the_native_backend(backend):
    with pytest.raises(ValueError):
        Model(4, 8, train_backend=backend, train_precision="tf32")


def test_state_dict_keys_unchanged():
    with open(os.path.join(HERE, "golden", "state_dict_surface.json")) as f:
        surface = json.load(f)
    sd = Model(train_precision="tf32").state_dict()
    assert [[k, list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd.items()] == surface["state_dict"]


def test_copies_keep_the_setting():
    m = Model(4, 8, train_precision="tf32")
    assert copy.deepcopy(m).train_precision == "tf32"
    assert pickle.loads(pickle.dumps(m)).train_precision == "tf32"


def _npad(c):
    """cols_of(c).npad of the tensor-core kernels: c in CTA tiles of up to four 16-column blocks, evenly filled"""
    b16 = -(-c // 16)
    ntiles = -(-b16 // 4)
    return -(-b16 // ntiles) * 16 * ntiles


def _floats(n):                                              # workspace regions are taken in 64-float (256-byte) units
    return -(-n // 64) * 64


def _packed_tf32(cout, cin, k):                              # [ceil(cin / 32) chunks][k taps][npad(cout) rows][32 channels]
    return -(-cin // 32) * k * _npad(cout) * 32


def _packed_bf16_floats(cout, cin, k):                       # bf16 [ceil(cin / 64)][k][npad(cout)][64], in floats
    return -(-(-(-cin // 64) * k * _npad(cout) * 64) // 2)


# (n_layers, channels_interval, B, T) -> workspace bytes of the fp32 and bf16 layouts, as the parent of this change gives them
LAYOUT_CASES = {(12, 24, 120, 16384): (5171055616, 5221651456), (12, 24, 2, 4096): (102267136, 152862976),
                (4, 8, 3, 256): (1043456, 1637376)}


@pytest.mark.parametrize("case", sorted(LAYOUT_CASES))
def test_tf32_layout_is_the_fp32_layout_plus_the_tf32_packings(case):
    n, ci, B, T = case
    fields = ("z", "act", "ga", "mean", "invstd", "s1", "s2", "Cin", "Cin0", "Cin1", "Cout", "L", "ksize", "mode")
    fp32 = [_lib.debug_train_layout(n, ci, B, T, i, "fp32") for i in range(2 * n + 1)]
    bf16 = [_lib.debug_train_layout(n, ci, B, T, i, "bf16") for i in range(2 * n + 1)]
    tf32 = [_lib.debug_train_layout(n, ci, B, T, i, "tf32") for i in range(2 * n + 1)]
    assert (fp32[0]["workspace_bytes"], bf16[0]["workspace_bytes"]) == LAYOUT_CASES[case]
    for a, t in zip(fp32, tf32):
        assert {f: a[f] for f in fields} == {f: t[f] for f in fields}
    extra_tf32 = sum(_floats(_packed_tf32(d["Cout"], d["Cin"], d["ksize"])) + _floats(_packed_tf32(d["Cin"], d["Cout"], d["ksize"]))
                     for d in fp32[1:])
    extra_bf16 = sum(_floats(_packed_bf16_floats(d["Cout"], d["Cin"], d["ksize"])) +
                     _floats(_packed_bf16_floats(d["Cin"], d["Cout"], d["ksize"])) for d in fp32[1:])
    assert tf32[0]["workspace_bytes"] == fp32[0]["workspace_bytes"] + 4 * extra_tf32
    assert bf16[0]["workspace_bytes"] == fp32[0]["workspace_bytes"] + 4 * extra_bf16
    for i, (b, t) in enumerate(zip(bf16, tf32)):
        assert t["workspace_bytes"] == tf32[0]["workspace_bytes"]
        if i == 0:                                           # block 0 (Cin = 1) stays on the fp32 weight gradient
            assert t["wgrad_tc"] == 0 and {k: t[k] for k in ("grid_x", "grid_y", "grid_z", "positions")} == \
                {k: fp32[0][k] for k in ("grid_x", "grid_y", "grid_z", "positions")}
            continue
        # the tf32 weight gradient has the bf16 one's CTA (64 co x 5 taps x 64 ci) and 64-position items
        assert t["wgrad_tc"] == 2 and b["wgrad_tc"] == 1
        assert {k: t[k] for k in ("grid_x", "grid_y", "grid_z", "items", "positions")} == \
            {k: b[k] for k in ("grid_x", "grid_y", "grid_z", "items", "positions")}


def test_layout_query_refuses_fp32_tc():
    with pytest.raises(_lib.WunetError):
        _lib.debug_train_layout(12, 24, 2, 4096, 0, "fp32_tc")


def test_inference_plan_query_refuses_tf32():
    buf = (ctypes.c_int * 32)()
    assert _lib.load().wunet_debug_plan_prec(12, 24, 2, 4096, 1, 132, buf, 32, _lib.PREC_TF32) == -1      # WUNET_EINVAL
