"""The tensor-core training convolutions (wunet_train_tc.cu: one source for bf16 and tf32, templated on the operand type) without a
GPU, kernel by kernel. The unit is compiled for sm_90a into a temporary directory (the in-tree library is untouched), and each
kernel's SASS and resource usage must be those recorded in tests/golden/train_tc_sass.json from the two per-precision units this
one replaced (tools/gen_train_tc_sass_golden.py): the merge changed no instruction, register, shared-memory or stack figure of
any of the 46 kernels. Keys name what a kernel computes (pass/precision/template arguments), not its mangled name. The ptxas
report of the same unit is checked by test_train_bf16_cpu.py."""
import json
import os
import sys

import pytest

from wave_u_net_for_speech_enhancement_b200 import build

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
import gen_train_tc_sass_golden as golden  # noqa: E402


def _nvcc():
    try:
        return build.nvcc_path()
    except RuntimeError:
        return None


with open(os.path.join(HERE, "golden", "train_tc_sass.json")) as _f:
    GOLDEN = json.load(_f)


@pytest.mark.skipif(not _nvcc() or golden.nvcc_release(_nvcc()) != GOLDEN["nvcc"],
                    reason=f"the recorded SASS is that of nvcc {GOLDEN['nvcc']}")
def test_train_tc_sass_is_the_recorded_sass(tmp_path):
    assert golden.NVCC_FLAGS == GOLDEN["flags"]
    obj = str(tmp_path / "wunet_train_tc.o")
    golden.compile_unit(_nvcc(), os.path.join(build.CSRC, "wunet_train_tc.cu"), obj)
    got, want = golden.kernels(_nvcc(), obj), GOLDEN["kernels"]
    assert sorted(got) == sorted(want) and len(want) == 46
    moved = [k for k in sorted(want) if got[k]["sass"] != want[k]["sass"]]
    assert not moved, f"SASS changed in {moved}; tools/gen_train_tc_sass_golden.py --dump writes it for a diff"
    res = {k: (got[k]["res"], want[k]["res"]) for k in sorted(want) if got[k]["res"] != want[k]["res"]}
    assert not res, f"resource usage changed (now, recorded): {res}"
