"""Half models without a GPU: the 16-bit I/O entry points and constants, the Python dtype dispatch and its refusals, the 16-bit
framing pass, and the inference units compiled for sm_90a. Those units are compiled once, in parallel, into a temporary directory
(the in-tree library is untouched): every float kernel must have the SASS and resource usage recorded in
tests/golden/forward_io_sass.json from the tree before the I/O type became a template argument
(tools/gen_forward_io_sass_golden.py). The 16-bit I/O forms (wunet_tc_io_*.cu, and the __half / __nv_bfloat16 instances in
wunet_fp32.cu) must compile without serialised wgmma and spill no more than their float forms (block 0's enc0_kernel keeps the
16-byte spill its float form has at 64 registers)."""
import concurrent.futures
import ctypes
import json
import os
import re
import sys

import numpy as np
import pytest
import torch

from wave_u_net_for_speech_enhancement_b200 import Model, _lib, build
from wave_u_net_for_speech_enhancement_b200.enhance import frame_clips

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tools"))
import gen_forward_io_sass_golden as golden  # noqa: E402

with open(os.path.join(HERE, "golden", "forward_io_sass.json")) as _f:
    GOLDEN = json.load(_f)

NEW = ["wunet_forward_io", "wunet_forward_host_io", "wunet_stream_submit_io", "wunet_frame_clips_f32_io", "wunet_frame_clips_i16_io"]


def _nvcc():
    try:
        return build.nvcc_path()
    except RuntimeError:
        return None


def test_io_symbols_and_constants():
    lib = _lib.load()
    for sym in NEW:
        assert sym in _lib.EXPORTED_SYMBOLS
        getattr(lib, sym)
    with open(os.path.join(os.path.dirname(HERE), "include", "wunet_b200.h")) as f:
        hdr = f.read()
    defs = dict(re.findall(r"#define (WUNET_IO_\w+) (\d+)", hdr))
    assert defs == {"WUNET_IO_F32": str(_lib.IO_F32), "WUNET_IO_F16": str(_lib.IO_F16), "WUNET_IO_BF16": str(_lib.IO_BF16)}
    assert (_lib.IO_F32, _lib.IO_F16, _lib.IO_BF16) == (0, 1, 2)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_dtype_dispatch(dtype):
    m = Model(4, 8).eval()
    x = torch.zeros(1, 1, 256)
    # float32 model: float32 input passes the checks (and stops at the missing device), 16-bit input is refused
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            m(x)
        with pytest.raises(RuntimeError, match=f"expected float32 input .* got {dtype}"):
            m(x.to(dtype))
    m.to(dtype)
    assert m._param_dtype() == dtype
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            m(x.to(dtype))                                    # accepted: the same dtype as the parameters
        name = str(dtype).replace("torch.", "")
        with pytest.raises(RuntimeError, match=f"expected {name} input .* got torch.float32"):
            m(x)
        with pytest.raises(RuntimeError, match=f"expected {name} input"):
            m.forward_host(x)
        assert m(x.to(dtype)[:0]).dtype == dtype               # an empty batch keeps the dtype
    m.out[0].bias.data = m.out[0].bias.data.float()           # mixed parameter dtypes
    assert m._param_dtype() is None
    with torch.no_grad(), pytest.raises(RuntimeError, match="mixed dtypes, got " + str(dtype)):
        m(x.to(dtype))
    m.to(dtype).train()
    with pytest.raises(RuntimeError, match="train_precision"):
        m(x.to(dtype))
    m.eval()
    with pytest.raises(RuntimeError, match="train_precision"):
        m(x.to(dtype).requires_grad_(True))


def test_half_state_dict_round_trip():
    m = Model(4, 8).half()
    sd = m.state_dict()
    other = Model(4, 8).half()
    other.load_state_dict(sd, strict=True)
    for k, v in other.state_dict().items():
        assert v.dtype == sd[k].dtype and torch.equal(v, sd[k])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_framing_rounds_once(dtype):
    rng = np.random.default_rng(3)
    clips_f = [rng.uniform(-1, 1, n).astype(np.float32) for n in (100, 16384 + 5, 0)]
    clips_i = [rng.integers(-32768, 32767, n, dtype=np.int16) for n in (100, 16384 + 5, 0)]
    for clips in (clips_f, clips_i):
        f32, index = frame_clips(clips, 256, pin=False, round_to=4)
        want = f32.clone().to(dtype)
        got, index16 = frame_clips(clips, 256, pin=False, round_to=4, dtype=dtype)
        assert index16 == index and got.dtype == dtype
        assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    with pytest.raises(_lib.WunetError, match="I/O dtype"):
        lens = (ctypes.c_longlong * 1)(4)
        buf = np.zeros(16, np.float32)
        _lib.check(_lib.load().wunet_frame_clips_f32_io((ctypes.c_void_p * 1)(buf.ctypes.data), lens, 1, 4, buf.ctypes.data, 4, 1, 7))


IO_UNITS = ["wunet_tc_io_f16.cu", "wunet_tc_io_bf16.cu"]     # the tensor-core forms with a 16-bit input / output (wunet_tc_io.cuh)


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    """{unit: (object path, nvcc output with the ptxas report)} of the inference units, compiled in parallel"""
    tmp = tmp_path_factory.mktemp("forward_io")

    def one(u):
        obj = str(tmp / u.replace(".cu", ".o"))
        return u, (obj, golden.sass.compile_unit(_nvcc(), os.path.join(build.CSRC, u), obj, ["-Xptxas", "-v"]))

    units = golden.UNITS + IO_UNITS
    with concurrent.futures.ThreadPoolExecutor(len(units)) as ex:
        return dict(ex.map(one, units))


needs_nvcc = pytest.mark.skipif(not _nvcc() or golden.sass.nvcc_release(_nvcc()) != GOLDEN["nvcc"],
                                reason=f"the recorded SASS is that of nvcc {GOLDEN['nvcc']}")


@needs_nvcc
def test_float_io_sass_is_the_recorded_sass(compiled):
    assert golden.sass.NVCC_FLAGS == GOLDEN["flags"]
    got = {}
    for u in golden.UNITS:
        obj = compiled[u][0]
        k = golden.sass.kernels(_nvcc(), obj, key_of=lambda d, u=u: golden.kernel_key(u, d) or "io16:" + d)
        got.update({key: v for key, v in k.items() if not key.startswith("io16:")})
    want = GOLDEN["kernels"]
    assert sorted(got) == sorted(want)
    moved = [k for k in sorted(want) if got[k]["sass"] != want[k]["sass"]]
    assert not moved, f"SASS changed in {moved}"
    res = {k: (got[k]["res"], want[k]["res"]) for k in sorted(want) if got[k]["res"] != want[k]["res"]}
    assert not res, f"resource usage changed (now, recorded): {res}"


@needs_nvcc
def test_io16_forms_spill_no_more_and_do_not_serialise_wgmma(compiled):
    forms = {}
    for u, (_obj, log) in compiled.items():
        bad = [line for line in log.splitlines() if re.search(r"C75(19|20)", line)]
        assert not bad, "\n".join(bad[:10])
        # ptxas reports each entry function, then its stack / spill line
        for name, body in re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'\n(.*?)(?=\nptxas info\s+: Compiling|\Z)", log, re.S):
            forms[(u, name)] = body
    demangled = golden.sass.demangle(_nvcc(), [n for _u, n in forms])
    # a demangled name without the return type template instances carry ("void ") and without the parameters
    name = lambda d: (d[5:] if d.startswith("void ") else d).split(">(")[0] + ">" if ">(" in d else d[:d.index("(")]  # noqa: E731
    io16 = {(u, n): body for (u, n), body in forms.items() if u in IO_UNITS or golden.kernel_key(u, demangled[n]) is None}
    names = " ".join(demangled[n] for _u, n in io16)
    # per I/O type: conv_tc_kernel heads (bf16: plain, merged tail, split; fp16: plain, merged tail), enc0_kernel (bf16, fp16),
    # x_to_bf16_kernel, enc0_wide_kernel (bf16, split, fp16), and the fp32 path's block 0 (two sliding-window forms, the generic
    # one) and out_kernel
    assert len(io16) == 2 * (3 + 2 + 2 + 1 + 3 + 4), sorted(demangled[n] for _u, n in io16)
    for form in ("conv_tc_kernel<", "enc0_kernel(", "enc0_wide_kernel<", "x_to_bf16_kernel(", "conv_slide_kernel<",
                 "conv_gen_kernel<", "out_kernel<"):
        assert form in names, form
    spill = lambda body: tuple(int(v) for v in re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", body).groups())  # noqa: E731

    def float_form(d):
        """the name of the float form of a 16-bit I/O kernel"""
        n = re.sub(r"(<|, )(__half|__nv_bfloat16)>", lambda m: "<float>" if m.group(1) == "<" else ", float>", name(d))
        n = n.replace("<float>", "").replace(", float>", ">")
        n = re.sub(r"^wunet::io_b?f16::", "wunet::", n)                 # wunet_tc_io.cuh's namespaces of the element types
        if "enc0_wide_kernel" in n:
            return n.replace("wunet::", "wunet::wide::", 1)
        return n.replace("wunet::bf16::", "wunet::")

    as_float = {golden.kernel_key("", demangled[n])[1:]: spill(b) for (u, n), b in forms.items() if (u, n) not in io16}
    more = {}
    for (u, n), b in io16.items():
        f = float_form(demangled[n])
        assert f in as_float, (demangled[n], f)
        if spill(b) > as_float[f]:
            more[demangled[n]] = (spill(b), as_float[f])
    assert not more, f"16-bit forms spilling more than their float forms (stores, loads): {more}"
