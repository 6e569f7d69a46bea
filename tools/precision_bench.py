"""Inference precisions side by side on one GPU: bf16, fp16 and fp32_tc at B x T (default 256 x 16384), legs alternated over
several repetitions, each leg timed with CUDA events over `--steps` forwards after `--warmup`. In the same run: the card, its
power limit and SM clock, the per-block times of bf16 against fp16 (Model.profile hooks), and, printed without asserting, the
max-abs error of fp16, bf16 and PyTorch eager (cuDNN TF32, the package's reference-semantics forward in eval mode) against the
fp32 native forward on the same weights and input. Writes JSON to --out if given.

    python tools/precision_bench.py [--batch 256] [--steps 100] [--warmup 5] [--reps 3] [--out precision.json]
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

LEGS = ("bf16", "fp16", "fp32_tc")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
        return r.stdout.strip()
    except OSError:
        return torch.cuda.get_device_name(0)


def model(prec, st):
    m = Model(12, 24, precision=prec)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()})
    return m.to("cuda:0").eval()


def time_leg(m, x, steps, warmup):
    with torch.no_grad():
        for _ in range(warmup):
            m(x)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            m(x)
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--T", type=int, default=16384)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("precision_bench needs a CUDA device")
    st = wo.make_state(12, 24, seed=0)
    x = torch.from_numpy(wo.make_input(a.batch, a.T, seed=1234)).cuda()
    models = {p: model(p, st) for p in LEGS}
    res = {"card": card(), "batch": a.batch, "T": a.T, "steps": a.steps, "warmup": a.warmup, "ms": {p: [] for p in LEGS}}
    print("card (name, power limit, SM clock, max SM clock):", res["card"])
    for rep in range(a.reps):
        for p in LEGS:
            ms = time_leg(models[p], x, a.steps, a.warmup)
            res["ms"][p].append(ms)
            print(f"rep {rep} {p:8s} {ms:7.3f} ms/forward  {a.batch * 1000.0 / ms:9.0f} frames/s")
    print("card after the timed legs:", card())
    for p in LEGS:
        best = min(res["ms"][p])
        print(f"{p:8s} best {best:7.3f} ms  {a.batch * 1000.0 / best:9.0f} frames/s  (all: {', '.join('%.3f' % v for v in res['ms'][p])})")
    r = min(res["ms"]["bf16"]) / min(res["ms"]["fp16"])
    print(f"fp16 frames/s / bf16 frames/s = {r:.4f}")
    # per-block device times, bf16 against fp16 (median of 20 profiled forwards)
    prof = {}
    with torch.no_grad():
        for p in ("bf16", "fp16"):
            m = models[p]
            m.profile(True)
            rows = []
            for _ in range(20):
                m(x)
                torch.cuda.synchronize()
                rows.append(m.profile_read())
            m.profile(False)
            prof[p] = np.median(np.array(rows), axis=0).tolist()
    res["per_block_ms"] = prof
    print("block   bf16 ms   fp16 ms   fp16/bf16")
    for i, (b, f) in enumerate(zip(prof["bf16"], prof["fp16"])):
        print(f"{i:5d} {b:9.4f} {f:9.4f} {f / b if b > 0 else float('nan'):9.3f}")
    # accuracy, printed only: against the native fp32 forward on the same weights and input (first 8 frames)
    xs = x[:8].contiguous()
    with torch.no_grad():
        ref = model("fp32", st)(xs)
        err = {p: float((models[p](xs) - ref).abs().max()) for p in ("fp16", "bf16")}
        torch.backends.cuda.matmul.allow_tf32 = True
        torch.backends.cudnn.allow_tf32 = True
        eager = models["fp16"]._forward_torch_reference_semantics(xs)
        err["eager_cudnn_tf32"] = float((eager - ref).abs().max())
    res["max_abs_vs_fp32"] = err
    print("max-abs vs the fp32 forward:", ", ".join(f"{k} {v:.2e}" for k, v in err.items()))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
