"""Wide channel plans side by side on one GPU: n_layers = 12, channels_interval 24 / 48 / 64, B x T (default 256 x 16384).
Legs: bf16, fp16, fp32_tc, precision="fp32" (CUDA-core FFMA) on the same weights and input, and PyTorch eager (cuDNN TF32, the
package's reference-semantics forward) for reference. The legs alternate over several repetitions; each is timed with CUDA
events over `--steps` forwards after `--warmup`. Max-abs errors against the fp32 leg are taken on the first 8 frames. The card,
its power limit and SM clock are printed in the same run. Writes JSON to --out if given.

    python tools/wide_plan_bench.py [--widths 24,48,64] [--batch 256] [--steps 10] [--warmup 2] [--reps 3] [--out wide.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import wunet_oracle as wo                                  # noqa: E402
from wave_u_net_for_speech_enhancement_b200 import Model               # noqa: E402

LEGS = ("bf16", "fp16", "fp32_tc", "fp32", "eager_cudnn_tf32")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
        return r.stdout.strip()
    except OSError:
        return torch.cuda.get_device_name(0)


def model(n, ci, prec, st):
    m = Model(n, ci, precision="fp32" if prec == "eager_cudnn_tf32" else prec)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()})
    return m.to("cuda:0").eval()


def forward(m, prec, x):
    if prec == "eager_cudnn_tf32":
        return m._forward_torch_reference_semantics(x)
    return m(x)


def time_leg(m, prec, x, steps, warmup):
    with torch.no_grad():
        for _ in range(warmup):
            forward(m, prec, x)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            forward(m, prec, x)
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--widths", default="24,48,64")
    ap.add_argument("--n", type=int, default=12)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--T", type=int, default=16384)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("wide_plan_bench needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    res = {"card": card(), "n": a.n, "batch": a.batch, "T": a.T, "steps": a.steps, "warmup": a.warmup, "widths": {}}
    print("card (name, power limit, SM clock, max SM clock):", res["card"])
    x = torch.from_numpy(wo.make_input(a.batch, a.T, seed=1234)).cuda()
    for ci in [int(v) for v in a.widths.split(",")]:
        st = wo.make_state(a.n, ci, seed=0)
        ms = {p: [] for p in LEGS}
        for rep in range(a.reps):
            for p in LEGS:                                          # one model alive at a time: the fp32 workspace is large
                m = model(a.n, ci, p, st)
                ms[p].append(time_leg(m, p, x, a.steps, a.warmup))
                m._release()
                del m
                torch.cuda.empty_cache()
                print(f"ci {ci} rep {rep} {p:17s} {ms[p][-1]:8.3f} ms/forward  {a.batch * 1000.0 / ms[p][-1]:9.0f} frames/s", flush=True)
        xs = x[:8].contiguous()
        with torch.no_grad():
            ref = model(a.n, ci, "fp32", st)(xs)
            err = {}
            for p in LEGS[:3] + LEGS[4:]:
                m = model(a.n, ci, p, st)
                err[p] = float((forward(m, p, xs) - ref).abs().max())
                m._release()
        best = {p: min(v) for p, v in ms.items()}
        res["widths"][ci] = {"ms": ms, "best_ms": best, "frames_per_s": {p: a.batch * 1000.0 / v for p, v in best.items()},
                             "max_abs_vs_fp32": err}
        print(f"ci {ci}: " + ", ".join(f"{p} {a.batch * 1000.0 / best[p]:.0f} f/s" for p in LEGS))
        print(f"ci {ci}: max-abs vs fp32 " + ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    print("card after the timed legs:", card())
    print("| ci | " + " | ".join(LEGS) + " | bf16 / fp32 |")
    for ci, r in res["widths"].items():
        f = r["frames_per_s"]
        print(f"| {ci} | " + " | ".join(f"{f[p] / 1000:.2f} k" for p in LEGS) + f" | {f['bf16'] / f['fp32']:.1f}x |")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fo:
            json.dump(res, fo, indent=1)


if __name__ == "__main__":
    main()
