"""The teacher-forced training check (tests/test_train_blocks_gpu.py) only means something if its cases reach the regimes where
the training kernels can go wrong. This guard reads its case table through the host-only layout query (no GPU needed):
every block's workspace regions are sound, and together the cases reach

- the fp32 weight gradient with >= 32 tiles per CTA (the tile loop) and with exactly one;
- the bf16, the tf32 and the fp16 weight gradient each with >= 100 items per CTA and with exactly one;
- a frame whose last 128-position (fp32) or 64-position (bf16, tf32) tile is partial;
- frames of fewer than 4 samples (the zero padding of the fp32 weight gradient's 4-position inner step);
- Cout not a multiple of 16 and Cin not a multiple of 64 (partial co / ci tiles), and a tf32 block whose Cin is not a
  multiple of 32 (a padded 32-channel K chunk of the tf32 forward);
- a block with Cin >= 1024 at fp32 and on the tensor cores at every tensor-core precision (the widest channel plans);
- B = 1, frozen BatchNorm, a backward without parameter gradients, and the part 0 / part 1 split (also at fp16_scaled, whose
  scale slots are cleared per part);
- the one-ulp replay of the middle block's BatchNorm backward reductions over >= 32768 values per channel, with frozen
  statistics, and at fp16_scaled (train_bn_bwd_apply_amax_kernel);
- a run with batch and frozen BatchNorm blocks side by side, and one whose backward stops early: null gradient slots below
  its lowest trainable block and no dx.

It fails as soon as a change of the case table or of the launch geometry drops one of them."""
import ctypes

import pytest

import test_train_blocks_gpu as blocks
from wave_u_net_for_speech_enhancement_b200 import _lib

REQUIRED = {"fp32_wgrad_ge_32_per_cta", "fp32_wgrad_1_per_cta", "bf16_wgrad_ge_100_per_cta", "bf16_wgrad_1_per_cta",
            "tf32_wgrad_ge_100_per_cta", "tf32_wgrad_1_per_cta", "tf32_cin_not_mult_32", "partial_tile", "frame_lt_4",
            "cout_not_mult_16", "cin_not_mult_64", "batch_1", "frozen", "no_param_grads", "part_split",
            "bn_reduction_ge_32768_per_channel", "bn_reduction_frozen",
            "fp16_wgrad_ge_100_per_cta", "fp16_wgrad_1_per_cta", "fp16_part_split", "fp16_bn_reduction", "cin_ge_1024",
            "fp32_cin_ge_1024", "mixed_bn_modes", "early_stop"}
FIELDS = ("z", "act", "ga", "mean", "invstd", "s1", "s2")
KIND = {0: "fp32", 1: "bf16", 2: "tf32", 3: "fp16"}      # wgrad_tc: the weight-gradient kernel of a block
TC_KINDS = ("bf16", "tf32", "fp16")


def regions(d, B):
    big = 4 * B * d["Cout"] * d["L"]
    return [(d[f], big if f in ("z", "act", "ga") else 4 * d["Cout"]) for f in FIELDS]


def layouts(case, prec):
    c = blocks.CASES[case]
    return [_lib.debug_train_layout(c["n"], c["ci"], c["B"], c["T"], i, prec) for i in range(2 * c["n"] + 1)]


def scale_slots(case, prec):
    """Field 22 of the layout query for every block: the byte offset of its fp16_scaled dz scale slot, -1 for none."""
    c = blocks.CASES[case]
    out = []
    for i in range(2 * c["n"] + 1):
        buf = (ctypes.c_longlong * 23)()
        _lib.check(_lib.load().wunet_debug_train_layout(c["n"], c["ci"], c["B"], c["T"], _lib.TRAIN_PRECISIONS[prec], i, buf, 23))
        out.append(buf[22])
    return out


@pytest.mark.parametrize("case", sorted(blocks.CASES))
def test_layout_regions_are_disjoint_aligned_and_inside_the_workspace(case):
    c = blocks.CASES[case]
    nb = 2 * c["n"] + 1
    for prec in ("fp32", "bf16", "tf32", "fp16_scaled"):
        lay = layouts(case, prec)
        total = lay[0]["workspace_bytes"]
        spans = []
        for i, d in enumerate(lay):
            assert d["workspace_bytes"] == total
            for off, size in regions(d, c["B"]):
                assert off % 256 == 0 and 0 <= off and off + size <= total, (case, prec, i, off, size, total)
                spans.append((off, off + size))
        slots = scale_slots(case, prec)
        if prec == "fp16_scaled":
            # 2n + 1 consecutive floats, block i's at base + 4 i; block 0 (fp32) reports none
            assert slots[0] == -1 and all(d["wgrad_tc"] == (0 if i == 0 else 3) for i, d in enumerate(lay)), case
            base = slots[1] - 4
            assert slots[1:] == [base + 4 * i for i in range(1, nb)], case
            assert base >= 0 and base % 4 == 0 and base + 4 * nb <= total, (case, base, total)
            spans += [(base + 4 * i, base + 4 * i + 4) for i in range(nb)]
        else:
            assert slots == [-1] * nb, (case, prec)
        spans.sort()
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])), (case, prec)
    fp32 = layouts(case, "fp32")
    for prec in ("bf16", "tf32", "fp16_scaled"):
        other = layouts(case, prec)
        for a, b in zip(fp32, other):
            assert {f: a[f] for f in FIELDS} == {f: b[f] for f in FIELDS}, (case, prec)
        assert fp32[0]["workspace_bytes"] <= other[0]["workspace_bytes"], (case, prec)


def test_layout_query_describes_the_channel_plan_and_the_weight_gradient_launch():
    n, ci, B, T = 12, 24, 120, 16384
    for prec in ("fp32", "bf16", "tf32"):
        for i in range(2 * n + 1):
            d = _lib.debug_train_layout(n, ci, B, T, i, prec)
            L = T >> i if i <= n else T >> (2 * n - i)
            assert (d["L"], d["ksize"], d["mode"]) == (L, 15 if i <= n else 5, 0 if i == 0 else 1 if i <= n else 2)
            assert d["Cin"] == d["Cin0"] + d["Cin1"] and (d["Cin1"] > 0) == (i > n)
            assert d["wgrad_tc"] == ({"fp32": 0, "bf16": 1, "tf32": 2}[prec] if i > 0 else 0)
            tiles = -(-L // d["positions"])
            assert d["items"] == B * tiles and d["items_per_cta"] == -(-d["items"] // d["grid_z"])
            if d["wgrad_tc"]:
                assert d["positions"] == 64 and d["grid_x"] == -(-d["Cout"] // 64) * (d["ksize"] // 5)
                if d["wgrad_tc"] == 2:
                    assert d["grid_y"] == -(-d["Cin"] // 64)
            else:
                assert d["positions"] == min(L, 128) and (d["grid_x"], d["grid_y"]) == (-(-d["Cout"] // 16), -(-d["Cin"] // 64))
    fp32 = [_lib.debug_train_layout(n, ci, B, T, i, "fp32")["items_per_cta"] for i in range(2 * n + 1)]
    bf16 = [_lib.debug_train_layout(n, ci, B, T, i, "bf16")["items_per_cta"] for i in range(1, 2 * n + 1)]
    tf32 = [_lib.debug_train_layout(n, ci, B, T, i, "tf32")["items_per_cta"] for i in range(1, 2 * n + 1)]
    assert (min(fp32), max(fp32), min(bf16), max(bf16)) == (4, 52, 14, 233)
    assert (min(tf32), max(tf32)) == (14, 233)                # dec11: 30720 items over 132 slices
    for bad in [(12, 24, 2, 4096, 25, "fp32"), (12, 24, 2, 4000, 0, "fp32"), (12, 24, 2, 4096, 0, "fp32_tc")]:
        with pytest.raises(_lib.WunetError):
            _lib.debug_train_layout(*bad)
    buf = (ctypes.c_longlong * 4)()
    assert _lib.load().wunet_debug_train_layout(12, 24, 2, 4096, _lib.PREC_FP32, 0, buf, 4) != 0


def features(case, prec, mode, pgrads):
    c = blocks.CASES[case]
    f = set()
    lay = layouts(case, prec)
    for d in lay:
        kind = KIND[d["wgrad_tc"]]
        if d["items_per_cta"] == 1:
            f.add(f"{kind}_wgrad_1_per_cta")
        if d["items_per_cta"] >= (32 if kind == "fp32" else 100):
            f.add(f"{kind}_wgrad_ge_{32 if kind == 'fp32' else 100}_per_cta")
        if kind == "tf32" and d["Cin"] % 32 != 0:
            f.add("tf32_cin_not_mult_32")
        if d["L"] % d["positions"] != 0:
            f.add("partial_tile")
        if d["L"] < 4:
            f.add("frame_lt_4")
        if d["Cout"] % 16 != 0:
            f.add("cout_not_mult_16")
        if d["Cin"] % 64 != 0:
            f.add("cin_not_mult_64")
        if d["Cin"] >= 1024:
            f.add(f"{kind}_cin_ge_1024")
    if c["B"] == 1:
        f.add("batch_1")
    if mode == "frozen":
        f.add("frozen")
    if not pgrads:
        f.add("no_param_grads")
    if mode == "blocks":
        frozen = set(c["bn_frozen"])
        if frozen and len(frozen) < len(lay):
            f.add("mixed_bn_modes")
        # the harness asks a "blocks" run for no dx: the backward stops at the lowest block with a gradient slot
        slots = [c["slots"].get(i, blocks.SLOTS) if pgrads else () for i in range(len(lay))]
        if not slots[0] and any(slots):
            f.add("early_stop")
    if (case, prec) in blocks.SPLIT:
        f |= {"part_split", "fp16_part_split"} if prec == "fp16_scaled" else {"part_split"}
    if (case, prec, mode, pgrads) in blocks.BN_REDUCTION:
        mid = lay[c["n"]]
        if c["B"] * mid["L"] >= 32768:
            f.add("bn_reduction_ge_32768_per_channel")
        if mode == "frozen":
            f.add("bn_reduction_frozen")
        if prec == "fp16_scaled":
            f.add("fp16_bn_reduction")
    return f


def test_bn_reduction_runs_are_runs_with_parameter_gradients():
    """The replay checks the BatchNorm parameter gradients, so every run it names must exist and compute them."""
    for r in blocks.BN_REDUCTION:
        assert r in blocks.RUNS and r[3], r


def test_cases_reach_every_training_regime():
    got = set()
    for case, prec, mode, pgrads in blocks.RUNS:
        got |= features(case, prec, mode, pgrads)
    if all(f"{k}_cin_ge_1024" in got for k in TC_KINDS):
        got.add("cin_ge_1024")                            # a tensor-core block with Cin >= 1024 at every tensor-core precision
    assert REQUIRED <= got, f"no case reaches {sorted(REQUIRED - got)}"
