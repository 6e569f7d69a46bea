"""Regenerate tests/golden/plan_n12_c24_b256.json from the library's host-side tiling decision (wunet_debug_plan).
Run after a tiling change has been validated on an H100 (GPU parity tests green with this plan)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from wave_u_net_for_speech_enhancement_b200 import _lib  # noqa: E402

KEYS = {"L": "L", "Cout": "Cout", "Nh": "Nh", "MT": "MT", "nacc": "nacc", "packed": "packed", "FR": "FR", "res": "resident",
        "bulk": "bulk_store", "na": "na", "nb": "nb", "tg": "tg", "smem": "smem", "tmem": "tmem_cols", "grid": "grid",
        "small": "small", "per_sm": "per_sm", "Cin0": "Cin0", "Cin1": "Cin1", "nsplit": "nsplit", "nchunks": "nchunks"}
blocks = []
for i in range(1, 25):
    d = _lib.debug_plan(12, 24, 256, 16384, i, 132)
    b = {k: d[v] for k, v in KEYS.items()}
    b["tiles"] = d["m_tiles"] * d["nsplit"]
    b["block"] = i
    blocks.append(b)
out = {"note": "tilings chosen by the library (wunet_debug_plan) for n_layers=12, channels_interval=24, B=256, T=16384 on 132 SMs "
               "(H100 SXM)",
       "num_sms": 132, "blocks": blocks}
json.dump(out, open(os.path.join(ROOT, "tests", "golden", "plan_n12_c24_b256.json"), "w"), indent=1)
print("wrote", len(blocks), "blocks")
