"""Model(train_precision=...) without a GPU: the constructor surface, and the training tensor-core kernels of wunet_train_tc.cu
(bf16 and tf32) compiled for sm_90a with ptxas in verbose mode (into a temporary directory, the in-tree library is untouched).
ptxas must report the conv and weight-gradient kernels and must not serialise their wgmma (C7520) or guard the accumulators
with extra warpgroup arrives (C7519), as test_wgmma_issue_cpu.py checks for wunet_tc.cu; test_train_tc_unit_cpu.py checks
the unit kernel by kernel."""
import copy
import json
import os
import pickle
import re
import subprocess

import pytest

from wave_u_net_for_speech_enhancement_b200 import Model, build

HERE = os.path.dirname(os.path.abspath(__file__))


def _nvcc():
    try:
        return build.nvcc_path()
    except RuntimeError:
        return None


@pytest.mark.skipif(_nvcc() is None, reason="needs nvcc")
def test_train_tc_kernels_compile_without_wgmma_serialisation(tmp_path):
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DWUNET_BUILD", "-Xptxas", "-v",
           "-c", os.path.join(build.CSRC, "wunet_train_tc.cu"), "-o", str(tmp_path / "wunet_train_tc.o")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = r.stdout + r.stderr
    assert r.returncode == 0, log[-4000:]
    assert "train_conv_tc_kernel" in log and "train_wgrad_tc_kernel" in log
    # the unit holds both precisions: per precision 16 convolutions, 6 weight gradients and 1 pack kernel
    entries = re.findall(r"Compiling entry function '(\w+)'", log)
    assert len(entries) == 46 and len([e for e in entries if "Tf32" in e or "tf32" in e]) == 23, entries
    assert "train_wgrad_tf32_kernel" in log
    bad = [line for line in log.splitlines() if re.search(r"C75(19|20)", line)]
    assert not bad, "\n".join(bad[:10])
    assert not re.search(r"[1-9]\d* bytes spill stores", log), "spills in the training tensor-core kernels"


def test_train_precision_default_is_fp32():
    assert Model(4, 8).train_precision == "fp32"
    assert Model(4, 8, train_precision="bf16").train_precision == "bf16"


@pytest.mark.parametrize("bad", ["fp16", "fp32_tc", "BF16", ""])
def test_bad_train_precision_raises(bad):
    with pytest.raises(ValueError):
        Model(4, 8, train_precision=bad)


@pytest.mark.parametrize("backend", ["torch", "none"])
def test_bf16_needs_the_native_backend(backend):
    with pytest.raises(ValueError):
        Model(4, 8, train_backend=backend, train_precision="bf16")
    assert Model(4, 8, train_backend=backend).train_precision == "fp32"


def test_state_dict_keys_unchanged():
    with open(os.path.join(HERE, "golden", "state_dict_surface.json")) as f:
        surface = json.load(f)
    sd = Model(train_precision="bf16").state_dict()
    assert [[k, list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd.items()] == surface["state_dict"]
    assert len(sd) == 177


def test_copies_keep_the_setting():
    m = Model(4, 8, train_precision="bf16")
    assert copy.deepcopy(m).train_precision == "bf16"
    assert pickle.loads(pickle.dumps(m)).train_precision == "bf16"
