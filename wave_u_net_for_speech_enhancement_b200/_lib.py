"""ctypes binding of libwunet_b200.so (the C ABI in include/wunet_b200.h). No torch types cross this boundary."""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("WUNET_LIB_PATH") or os.path.join(_HERE, "libwunet_b200.so")   # env: development builds (tracing)

PREC_FP32 = 0
PREC_BF16 = 1
PREC_FP32_TC = 2
PREC_TF32 = 3
PREC_FP16 = 4
PREC_FP16_SCALED = 5
PRECISIONS = {"fp32": PREC_FP32, "bf16": PREC_BF16, "fp32_tc": PREC_FP32_TC, "fp16": PREC_FP16}   # inference (Model(precision=...))
TRAIN_PRECISIONS = {"fp32": PREC_FP32, "bf16": PREC_BF16, "tf32": PREC_TF32,      # training step (Model(train_precision=...))
                    "fp16_scaled": PREC_FP16_SCALED}

IO_F32 = 0                 # element type of the network input / output (the _io entry points)
IO_F16 = 1
IO_BF16 = 2

TRAIN_FROZEN_BN = 1        # training-step flags (include/wunet_b200.h): eval-mode BatchNorm
TRAIN_NO_PARAM_GRADS = 2   # backward: input gradient only
TRAIN_DETERMINISTIC = 16   # bitwise repeatable step (no float atomics; larger workspace)

# wunet_bn_allreduce_fn(user, buf, count, stream): sums buf[0 .. count) (device doubles) over the ranks, ordered on stream
BN_ALLREDUCE_FN = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p)

_lib = None


class WunetError(RuntimeError):
    """Raised when a libwunet_b200 call returns a negative status (message from wunet_last_error())."""


def load() -> ctypes.CDLL:
    """Load the CUDA library; there is deliberately no fallback if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise ImportError(
            f"{SO_PATH} is missing: build it with `python -m wave_u_net_for_speech_enhancement_b200.build` "
            "(needs nvcc; sm_90a only). This package has no CPU / PyTorch fallback for the forward path.")
    lib = ctypes.CDLL(SO_PATH)
    vp, ci, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    lib.wunet_version.restype = ctypes.c_char_p
    lib.wunet_last_error.restype = ctypes.c_char_p
    lib.wunet_create.argtypes = [ci, ci, ci, ctypes.POINTER(vp)]
    lib.wunet_destroy.argtypes = [vp]
    lib.wunet_destroy.restype = None
    lib.wunet_num_blocks.argtypes = [vp]
    lib.wunet_block_shape.argtypes = [vp, ci, ctypes.POINTER(ci), ctypes.POINTER(ci), ctypes.POINTER(ci)]
    lib.wunet_set_weights.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.wunet_workspace_bytes.argtypes = [vp, ci, ci, ci]
    lib.wunet_workspace_bytes.restype = cs
    lib.wunet_forward.argtypes = [vp, vp, vp, ci, ci, ci, vp, cs, vp]
    lib.wunet_forward_host.argtypes = [vp, vp, vp, ci, ci, ci]
    lib.wunet_stream_submit.argtypes = [vp, vp, vp, ci, ci, ci, ctypes.POINTER(ci)]
    lib.wunet_stream_wait.argtypes = [vp, ci]
    lib.wunet_forward_io.argtypes = [vp, vp, vp, ci, ci, ci, ci, vp, cs, vp]
    lib.wunet_forward_host_io.argtypes = [vp, vp, vp, ci, ci, ci, ci]
    lib.wunet_stream_submit_io.argtypes = [vp, vp, vp, ci, ci, ci, ci, ctypes.POINTER(ci)]
    lib.wunet_read_level.argtypes = [vp, ci, vp, ci, ci, ci, vp, vp]
    lib.wunet_forward_export.argtypes = [vp, vp, vp, ci, ci, ci, ci, vp, vp, vp, cs, vp]
    ll = ctypes.c_longlong
    lib.wunet_frame_clips_f32.argtypes = [vp, vp, ci, ci, vp, ll, ci]
    lib.wunet_frame_clips_i16.argtypes = [vp, vp, ci, ci, vp, ll, ci]
    lib.wunet_unframe_clips_f32.argtypes = [vp, vp, vp, ci, ci, ll, ci]
    lib.wunet_frame_clips_f32_io.argtypes = [vp, vp, ci, ci, vp, ll, ci, ci]
    lib.wunet_frame_clips_i16_io.argtypes = [vp, vp, ci, ci, vp, ll, ci, ci]
    lib.wunet_wav_info.argtypes = [ctypes.c_char_p, ctypes.POINTER(ci), ctypes.POINTER(ci), ctypes.POINTER(ll), ctypes.POINTER(ci), ctypes.POINTER(ci)]
    lib.wunet_wav_read_f32.argtypes = [ctypes.c_char_p, ll, ll, vp]
    lib.wunet_crop_pairs.argtypes = [vp, vp, vp, vp, ci, ci, ci, vp, vp, ci]
    lib.wunet_last_launch_count.argtypes = [vp]
    lib.wunet_profile_enable.argtypes = [vp, ci]
    lib.wunet_profile_read.argtypes = [vp, vp, ci, ctypes.POINTER(ci)]
    lib.wunet_debug_plan.argtypes = [ci, ci, ci, ci, ci, ci, ctypes.POINTER(ci), ci]
    lib.wunet_debug_plan_prec.argtypes = lib.wunet_debug_plan.argtypes + [ci]
    lib.wunet_debug_plan_m2.argtypes = lib.wunet_debug_plan_prec.argtypes
    lib.wunet_debug_pair_weights.argtypes = [vp, ci, ci, ci, ci, ci, vp]
    lib.wunet_train_workspace_bytes.argtypes = [vp, ci, ci]
    lib.wunet_train_workspace_bytes.restype = cs
    lib.wunet_train_forward.argtypes = [vp, vp, vp, ci, ci, vp, vp, vp, vp, vp, vp, vp, vp, ctypes.c_float, vp, cs, vp]
    lib.wunet_train_backward.argtypes = [vp, vp, vp, vp, ci, ci, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, cs, vp]
    lib.wunet_train_backward_part.argtypes = [vp, vp, vp, vp, ci, ci, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, cs, vp, ci]
    lib.wunet_train_workspace_bytes_prec.argtypes = [vp, ci, ci, ci]
    lib.wunet_train_workspace_bytes_prec.restype = cs
    lib.wunet_train_workspace_bytes_ex.argtypes = [vp, ci, ci, ci, ci]
    lib.wunet_train_workspace_bytes_ex.restype = cs
    lib.wunet_train_forward_prec.argtypes = lib.wunet_train_forward.argtypes + [ci]
    lib.wunet_train_backward_part_prec.argtypes = lib.wunet_train_backward_part.argtypes + [ci]
    lib.wunet_train_forward_ex.argtypes = lib.wunet_train_forward_prec.argtypes + [ci]
    lib.wunet_train_backward_ex.argtypes = lib.wunet_train_backward.argtypes + [vp, ci, ci, ci]
    lib.wunet_train_forward_blocks.argtypes = lib.wunet_train_forward_ex.argtypes + [vp, vp]
    lib.wunet_train_backward_blocks.argtypes = lib.wunet_train_backward_ex.argtypes + [vp]
    lib.wunet_train_backward_inject.argtypes = lib.wunet_train_backward_blocks.argtypes + [vp]
    lib.wunet_train_set_bn_allreduce.argtypes = [vp, BN_ALLREDUCE_FN, vp, vp, cs]
    lib.wunet_debug_train_conv.argtypes = [ci, ci, ci, ci, ci, ci, ci, ci, ci, vp, vp, vp, vp, vp]
    lib.wunet_debug_train_layout.argtypes = [ci, ci, ci, ci, ci, ci, ctypes.POINTER(ll), ci]
    lib.wunet_debug_train_dz_scale.argtypes = [ctypes.c_float]
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        raise WunetError(f"libwunet_b200: {load().wunet_last_error().decode()} (status {rc})")


EXPORTED_SYMBOLS = [
    "wunet_version", "wunet_last_error", "wunet_create", "wunet_destroy", "wunet_num_blocks", "wunet_block_shape",
    "wunet_set_weights", "wunet_workspace_bytes", "wunet_forward", "wunet_forward_host", "wunet_stream_submit", "wunet_stream_wait", "wunet_read_level",
    "wunet_last_launch_count", "wunet_profile_enable", "wunet_profile_read", "wunet_debug_plan", "wunet_debug_plan_prec",
    "wunet_debug_pair_weights",
    "wunet_train_workspace_bytes", "wunet_train_forward", "wunet_train_backward", "wunet_train_backward_part",
    "wunet_train_workspace_bytes_prec", "wunet_train_forward_prec", "wunet_train_backward_part_prec", "wunet_debug_train_conv",
    "wunet_train_forward_ex", "wunet_train_backward_ex", "wunet_train_workspace_bytes_ex", "wunet_debug_train_layout",
    "wunet_train_set_bn_allreduce", "wunet_train_forward_blocks", "wunet_train_backward_blocks", "wunet_debug_train_dz_scale",
    "wunet_frame_clips_f32", "wunet_frame_clips_i16", "wunet_unframe_clips_f32",
    "wunet_wav_info", "wunet_wav_read_f32", "wunet_crop_pairs",
    "wunet_forward_io", "wunet_forward_host_io", "wunet_stream_submit_io", "wunet_frame_clips_f32_io", "wunet_frame_clips_i16_io",
    "wunet_forward_export", "wunet_train_backward_inject", "wunet_debug_plan_m2",
]

PLAN_FIELDS = ["L", "Cin0", "Cin1", "Cout", "Npad", "Nh", "nsplit", "Nstride", "MT", "nacc", "packed", "FR", "S", "m_tiles",
               "nchunks", "resident", "bulk_store", "na", "nb", "tg", "ngroups", "a_stage_bytes", "b_stage_bytes", "a_tx_bytes",
               "rows_used", "tmem_cols", "smem", "threads", "per_sm", "grid", "small", "tiles_per_frame"]


def debug_plan(n_layers: int, channels_interval: int, B: int, T: int, block: int, num_sms: int = 148,
               precision: str = "bf16") -> dict:
    """The tiling the bf16 (or fp32_tc) path would choose for one conv block (host-only query: works without a GPU)."""
    buf = (ctypes.c_int * 32)()
    check(load().wunet_debug_plan_prec(n_layers, channels_interval, B, T, block, num_sms, buf, 32, PRECISIONS[precision]))
    return dict(zip(PLAN_FIELDS, [int(v) for v in buf]))


M2_FIELDS = ["selected", "na", "nb", "tg", "ngroups", "smem", "grid", "units"]


def debug_plan_m2(n_layers: int, channels_interval: int, B: int, T: int, block: int, num_sms: int = 148,
                  precision: str = "bf16") -> dict:
    """Whether one conv block runs in 256-row units (two tiles per unit, each weight stage serving both) and the geometry of
    that form; all zero when it does not (host-only query: works without a GPU)."""
    buf = (ctypes.c_int * len(M2_FIELDS))()
    check(load().wunet_debug_plan_m2(n_layers, channels_interval, B, T, block, num_sms, buf, len(M2_FIELDS), PRECISIONS[precision]))
    return dict(zip(M2_FIELDS, [int(v) for v in buf]))


TRAIN_LAYOUT_FIELDS = ["z", "act", "ga", "mean", "invstd", "s1", "s2", "Cin", "Cin0", "Cin1", "Cout", "L", "ksize", "mode",
                       "wgrad_tc", "grid_x", "grid_y", "grid_z", "items", "positions", "items_per_cta", "workspace_bytes"]


def debug_train_layout(n_layers: int, channels_interval: int, B: int, T: int, block: int, precision: str = "fp32") -> dict:
    """Where one block's tensors live in the training workspace (byte offsets) and how its weight gradient is launched
    (host-only query: works without a GPU)."""
    n = len(TRAIN_LAYOUT_FIELDS)
    buf = (ctypes.c_longlong * n)()
    code = TRAIN_PRECISIONS[precision] if precision in TRAIN_PRECISIONS else PRECISIONS[precision]   # fp32_tc: refused by the library
    check(load().wunet_debug_train_layout(n_layers, channels_interval, B, T, code, block, buf, n))
    return dict(zip(TRAIN_LAYOUT_FIELDS, [int(v) for v in buf]))
