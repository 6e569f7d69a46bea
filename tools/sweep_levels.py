"""Per-block tiling sweep of the bf16 path (development tool, needs the GPU).

    python tools/sweep_levels.py --journal gpurun_out/sweep.jsonl [--blocks 7,8] [--batch 256]

Every candidate is one WUNET_TC_OVR override of ONE block (see wunet_tc.cu: parse_override); the block's device time
comes from the library's per-block events (wunet_profile_*), the output is compared with the default plan's output
(the accumulation order does not depend on the tiling, so the comparison is exact). The journal makes the sweep
resumable: a candidate that crashed or hung the process is skipped on the next start.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import wunet_oracle as wo  # noqa: E402
from wave_u_net_for_speech_enhancement_b200 import Model  # noqa: E402

N, CI, T = 12, 24, 16384


def block_shape(i):
    L = (T >> i) if i <= N else (T >> (2 * N - i))
    cout = (i + 1) * CI if i < N else (N * CI if i == N else (2 * N - i + 1) * CI)
    return L, cout


def candidates(i):
    L, cout = block_shape(i)
    dec = i > N
    out = []
    if L < 128:
        for small in (0, 1):
            for mt in (1, 2, 3, 4):
                for ns in (1, 2, 3, 4, 6):
                    out.append(f"{i}:mt={mt},ns={ns},small={small}")
    else:
        mts = [m for m in (1, 2, 3, 4) if 128 * m <= L]
        for small in (0, 1):
            for mt in mts:
                for ns in (1, 2):
                    out.append(f"{i}:mt={mt},ns={ns},small={small}")
                    if dec:
                        out.append(f"{i}:mt={mt},ns={ns},small={small},na=3")
                    if mt <= 2:
                        out.append(f"{i}:mt={mt},ns={ns},small={small},nacc=1")
        if L == 128:
            for small in (0, 1):
                for mt in (2, 3, 4):
                    for ns in (1, 2, 3):
                        out.append(f"{i}:packed=1,mt={mt},ns={ns},small={small}")
    return out


def measure(m, x, reps):
    with torch.no_grad():
        y = m(x)
        tot = None
        for _ in range(reps):
            y = m(x)
            ms = np.array(m.profile_read())
            tot = ms if tot is None else tot + ms
    torch.cuda.synchronize()
    return y, tot / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--journal", default=os.path.join(ROOT, "gpurun_out", "sweep.jsonl"))
    ap.add_argument("--blocks", default="")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--combine", action="store_true", help="after the sweep, time the per-block winners together")
    args = ap.parse_args()
    blocks = [int(b) for b in args.blocks.split(",") if b] or list(range(1, 2 * N + 1))

    started = set()
    results = []
    if os.path.exists(args.journal):
        for line in open(args.journal):
            try:
                r = json.loads(line)
            except ValueError:
                continue
            if r.get("ev") == "start":
                started.add(r["cfg"])
            elif r.get("ev") == "done":
                results.append(r)
    jf = open(args.journal, "a")

    def log(**kw):
        jf.write(json.dumps(kw) + "\n")
        jf.flush()
        os.fsync(jf.fileno())

    st = wo.make_state(N, CI, seed=0)
    m = Model(N, CI, precision="bf16")
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()})
    m = m.cuda().eval()
    x = torch.from_numpy(wo.make_input(args.batch, T, seed=1)).cuda()
    os.environ.pop("WUNET_TC_OVR", None)
    with torch.no_grad():
        m(x)
    m.profile(True)
    y_ref, base = measure(m, x, 8)
    y_ref = y_ref.clone()
    print("baseline ms/forward %.4f" % base.sum(), flush=True)
    log(ev="base", ms=[float(v) for v in base])

    for i in blocks:
        for cfg in candidates(i):
            if cfg in started:
                continue
            log(ev="start", cfg=cfg)
            os.environ["WUNET_TC_OVR"] = cfg
            try:
                y, ms = measure(m, x, args.reps)
                diff = float((y - y_ref).abs().max())
                r = dict(ev="done", cfg=cfg, block=i, us=float(ms[i]) * 1e3, base_us=float(base[i]) * 1e3, diff=diff)
            except Exception as e:  # plan rejected (does not fit / illegal tiling) ... or the context died
                try:
                    torch.zeros(1, device="cuda").add_(1)
                    torch.cuda.synchronize()
                except Exception:
                    print("context lost at %s: %s" % (cfg, str(e)[:200]), flush=True)
                    os._exit(3)
                r = dict(ev="done", cfg=cfg, block=i, err=str(e)[:120])
            log(**r)
            results.append(r)
            if "us" in r:
                print("%-44s %8.1f us (base %8.1f)  diff %.1e" % (cfg, r["us"], r["base_us"], r["diff"]), flush=True)
    os.environ.pop("WUNET_TC_OVR", None)

    best = {}
    for r in results:
        if "us" not in r or r["diff"] != 0.0:
            continue
        b = r["block"]
        if r["us"] < 0.97 * r["base_us"] and (b not in best or r["us"] < best[b]["us"]):
            best[b] = r
    print("---- winners (>3 %% faster than the default plan, exact output)")
    for b in sorted(best):
        print("%-44s %8.1f us (base %8.1f)" % (best[b]["cfg"], best[b]["us"], best[b]["base_us"]))
    if args.combine and best:
        combo = ";".join(best[b]["cfg"] for b in sorted(best))
        os.environ["WUNET_TC_OVR"] = combo
        y, ms = measure(m, x, 10)
        print("combined: %.4f ms/forward (default %.4f), diff %.1e" % (ms.sum(), base.sum(), float((y - y_ref).abs().max())))
        print("WUNET_TC_OVR=" + combo)
        log(ev="combo", cfg=combo, ms=float(ms.sum()), base=float(base.sum()))
    m._release()


if __name__ == "__main__":
    main()
