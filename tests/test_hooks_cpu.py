"""Forward hooks on the block containers, without a GPU: the new C entry points are exported, the hook scan fires on exactly
the supported containers and refuses every other sub-module hook with an error naming the module (before the device check,
so the refusals are the same on the CPU), and the unit holding the hooks' kernels compiles for sm_90a without spills."""
import os
import re
import subprocess

import pytest
import torch

from wave_u_net_for_speech_enhancement_b200 import Model, _lib
from wave_u_net_for_speech_enhancement_b200 import build as wbuild


def test_entry_points_are_exported():
    lib = _lib.load()
    for sym in ("wunet_forward_export", "wunet_train_backward_inject"):
        assert sym in _lib.EXPORTED_SYMBOLS
        getattr(lib, sym)


def model(n=4, ci=8, **kw):
    return Model(n, ci, precision="fp32", **kw)


def x_of(T=256):
    return torch.zeros(2, 1, T)


def test_no_hook_means_no_plan_and_a_cached_scan():
    m = model()
    assert m._forward_hook_plan() is None
    assert m._hook_free_at is not None
    h = m.decoder[3].register_forward_hook(lambda *a: None)       # a new handle invalidates the cached scan
    plan = m._forward_hook_plan()
    assert [p[0] for p in plan] == ["decoder.3"]
    h.remove()
    assert m._forward_hook_plan() is None


def test_plan_order_and_levels():
    m = model()
    hs = [mod.register_forward_hook(lambda *a: None) for mod in (m.out, m.middle, m.encoder[1].main, m.decoder[0], m.encoder[1])]
    plan = m._forward_hook_plan()
    assert [p[0] for p in plan] == ["encoder.1.main", "encoder.1", "middle", "decoder.0", "out"]
    # outputs, the inputs' sources (encoder 0 for encoder 1, encoder 3 for the middle, middle + encoder 3 for decoder 0) and
    # the last decoder for the head's input
    assert m._hook_levels(plan) == [0, 1, 3, 4, 5, 8]
    for h in hs:
        h.remove()


def test_global_forward_hook_selects_every_container():
    m = model()
    h = torch.nn.modules.module.register_module_forward_hook(lambda *a: None)
    try:
        plan = m._forward_hook_plan()
    finally:
        h.remove()
    assert len(plan) == 2 * 4 + 2 * 4 + 2
    assert m._hook_levels(plan) == list(range(9))


@pytest.mark.parametrize("train", [False, True])
@pytest.mark.parametrize("target,register,exc", [
    ("decoder.1", lambda m: m.decoder[1].register_forward_pre_hook(lambda *a: None), NotImplementedError),
    ("encoder.0.main", lambda m: m.encoder[0].main.register_forward_pre_hook(lambda *a: None), NotImplementedError),
    ("encoder.2.main.0", lambda m: m.encoder[2].main[0].register_forward_hook(lambda *a: None), NotImplementedError),
    ("middle.1", lambda m: m.middle[1].register_forward_hook(lambda *a: None), NotImplementedError),
    ("decoder.3.main.2", lambda m: m.decoder[3].main[2].register_forward_hook(lambda *a: None), NotImplementedError),
    ("out.1", lambda m: m.out[1].register_forward_hook(lambda *a: None), NotImplementedError),
    ("middle", lambda m: m.middle.register_full_backward_hook(lambda *a: None), NotImplementedError),
    ("encoder.3", lambda m: m.encoder[3].register_full_backward_pre_hook(lambda *a: None), NotImplementedError),
    ("out.0", lambda m: m.out[0].register_full_backward_hook(lambda *a: None), NotImplementedError),
])
def test_refusals_name_the_module(train, target, register, exc):
    m = model().train(train)
    h = register(m)
    with pytest.raises(exc, match=re.escape(target) + r" \("):
        m(x_of())
    h.remove()


def test_a_hook_returning_a_value_is_refused():
    m = model().eval()
    m.encoder[2].register_forward_hook(lambda mod, a, o: o)
    # an empty batch fires the hooks without the device (the reference returns an empty batch, so do we)
    with pytest.raises(RuntimeError, match=r"encoder\.2 \(DownSamplingLayer\) returned a value"):
        m(torch.zeros(0, 1, 256))


def test_empty_batch_fires_hooks_with_empty_levels():
    m = model().eval()
    seen = []
    for mod in (m.encoder[0], m.middle, m.decoder[3], m.out):
        mod.register_forward_hook(lambda mod, a, o: seen.append((tuple(a[0].shape), tuple(o.shape))))
    kw_seen = []
    m.decoder[0].register_forward_hook(lambda mod, a, kw, o: kw_seen.append(kw), with_kwargs=True)
    m(torch.zeros(0, 1, 256))
    assert seen == [((0, 1, 256), (0, 8, 256)), ((0, 32, 16), (0, 32, 16)), ((0, 24, 256), (0, 8, 256)), ((0, 9, 256), (0, 1, 256))]
    assert kw_seen == [{}]


def test_torch_backend_keeps_real_module_hooks():
    """The composite path calls the sub-modules: its hooks (pre-hooks and inner modules included) behave as in torch."""
    m = model(train_backend="torch").train()
    seen = []
    m.encoder[0].main[0].register_forward_pre_hook(lambda mod, a: seen.append("pre"))
    m(torch.randn(2, 1, 256))
    assert seen == ["pre"]


def test_hooks_unit_compiles_without_spills(tmp_path):
    src = os.path.join(wbuild.CSRC, "wunet_hooks.cu")
    cmd = [wbuild.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
           "-DWUNET_BUILD", "-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "wunet_hooks.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    log = out.stdout + out.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) >= 7 and all(s == ("0", "0") for s in spills), log
    assert "C7519" not in log and "C7520" not in log
