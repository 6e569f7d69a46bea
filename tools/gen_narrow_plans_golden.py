"""Record tests/golden/plans_narrow.json: the tensor-core plans (wunet_debug_plan) of every channel plan up to 32 base filters
that tests/test_plan_cpu.py::test_plan_invariants covers, at its batches and lengths, for bf16, fp16 and fp32_tc on 132 SMs.

The wide-plan change (channels_interval 40 .. 64) must leave these plans field for field as they were, so the golden is recorded
from the library of the commit before it:
    git worktree add /tmp/parent <commit>; (cd /tmp/parent && python -m wave_u_net_for_speech_enhancement_b200.build)
    python tools/gen_narrow_plans_golden.py --lib-root /tmp/parent
The 6,624 plans (32 fields each, or the refusal message) are stored as one sha256 per (n_layers, channels_interval, precision)
over their canonical JSON, with the plan count: the test names the group that moved, and `--dump` writes the plans themselves
for a diff against the same dump of another library."""
import argparse
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [(4, 8), (8, 16), (12, 24), (12, 32), (12, 8), (10, 24)]         # test_plan_invariants' (n, ci) ...
BATCHES = [1, 2, 3, 17, 64, 128, 256, 1000]                              # ... its batches
PRECISIONS = ["bf16", "fp16", "fp32_tc"]
SMS = 132


def lengths(n):
    return sorted({1 << n, 4 << n, 16384 if 16384 % (1 << n) == 0 else 8 << n})     # test_plan_invariants' T values


def record(lib):
    """{"n,ci,B,T,block,precision": [32 values] or "error: <message>"}"""
    plans = {}
    for n, ci in CASES:
        for B in BATCHES:
            for T in lengths(n):
                for i in range(1, 2 * n + 1):
                    for prec in PRECISIONS:
                        key = f"{n},{ci},{B},{T},{i},{prec}"
                        try:
                            d = lib.debug_plan(n, ci, B, T, i, SMS, precision=prec)
                            plans[key] = [d[f] for f in lib.PLAN_FIELDS]
                        except lib.WunetError as e:
                            plans[key] = "error: " + str(e)
    return plans


def digests(plans):
    """{"n,ci,precision": {"plans": count, "sha256": digest of the group's plans in canonical JSON (sorted keys)}}"""
    groups = {}
    for key, v in plans.items():
        n, ci, _, _, _, prec = key.split(",")
        groups.setdefault(f"{n},{ci},{prec}", {})[key] = v
    return {g: {"plans": len(p), "sha256": hashlib.sha256(json.dumps(p, sort_keys=True, separators=(",", ":")).encode()).hexdigest()}
            for g, p in groups.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--lib-root", default=ROOT, help="checkout whose built library answers the queries")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "plans_narrow.json"))
    ap.add_argument("--dump", default=None, help="also write every plan to this file (for diffing two libraries)")
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.lib_root))
    from wave_u_net_for_speech_enhancement_b200 import _lib
    assert os.path.abspath(_lib.__file__).startswith(os.path.abspath(a.lib_root)), _lib.__file__
    plans = record(_lib)
    if a.dump:
        with open(a.dump, "w") as f:
            json.dump({"fields": list(_lib.PLAN_FIELDS), "plans": plans}, f, separators=(",", ":"))
    g = {"note": f"wunet_debug_plan at {SMS} SMs (H100 SXM) for test_plan_invariants' channel plans, batches and lengths: one "
                 "sha256 per (n_layers, channels_interval, precision) over the canonical JSON of its plans (tools/gen_narrow_plans_golden.py)",
         "num_sms": SMS, "fields": list(_lib.PLAN_FIELDS), "groups": digests(plans)}
    with open(a.out, "w") as f:
        json.dump(g, f, indent=1)
        f.write("\n")
    print("wrote", len(g["groups"]), "group digests over", len(plans), "plans to", a.out)


if __name__ == "__main__":
    main()
