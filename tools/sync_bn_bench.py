"""Cost of synchronised BatchNorm statistics in the native training step (reference architecture, n_layers 12,
channels_interval 24, T = 16384), one GPU, two legs per training precision:

    default       Model(train_precision=p): per-rank BatchNorm statistics (the step's usual launches)
    passthrough   the same model with a pass-through BatchNorm all-reduce hook (``model._bn_allreduce`` returning at once):
                  the split statistics kernels and the 75 host callbacks per step (2 per block in the forward, 1 per block
                  in the backward), with no communication. What a world of one rank would add; the cross-rank collectives
                  themselves are not in it.

Each step is what trainer/trainer.py:34-38 does: forward, MSE loss, backward, Adam (lr 1e-3). Per (B, precision) both legs run
`--warmup` untimed steps, then `--steps` timed ones alternately over `--reps` repetitions; CUDA events around the whole step
give the device time, and a host clock around each timed window (ending in a device synchronise) is reported beside it. The
GPU name, power limit and SM clocks are read with nvidia-smi in the same run. Writes sync_bn_bench.json into --out.

    python tools/sync_bn_bench.py --out /tmp/sbb                        # B = 64 and 120, fp32 and bf16
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from train_precision_bench import gpu_info  # noqa: E402
from wave_u_net_for_speech_enhancement_b200 import Model  # noqa: E402

LEGS = ("default", "passthrough")


def make_leg(leg, prec, B, T):
    torch.manual_seed(0)
    m = Model(12, 24, precision="fp32", train_precision=prec).cuda().train()
    calls = []
    if leg == "passthrough":
        m._bn_allreduce = lambda buf: calls.append(1)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, betas=(0.9, 0.999))
    g = torch.Generator(device="cuda").manual_seed(1)
    clean = 0.1 * torch.randn(B, 1, T, device="cuda", generator=g)
    noisy = clean + 0.05 * torch.randn(B, 1, T, device="cuda", generator=g)
    return m, opt, noisy, clean, calls


def run_steps(state, n):
    m, opt, noisy, clean, calls = state
    crit = torch.nn.MSELoss()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    torch.cuda.synchronize()
    c0, t0 = len(calls), time.perf_counter()
    for e in ev:
        e[0].record()
        opt.zero_grad()
        crit(clean, m(noisy)).backward()                   # trainer/trainer.py:36 argument order
        opt.step()
        e[1].record()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return {"step_ms": float(np.mean([a.elapsed_time(b) for a, b in ev])), "wall_step_ms": 1e3 * wall / n,
            "hook_calls_per_step": (len(calls) - c0) / n}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True, help="output directory (sync_bn_bench.json)")
    ap.add_argument("--batches", default="64,120")
    ap.add_argument("--precisions", default="fp32,bf16")
    ap.add_argument("--T", type=int, default=16384)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sync_bn_bench: needs a CUDA device (no CPU measurement)")
    os.makedirs(a.out, exist_ok=True)
    result = {"gpu_before": gpu_info(), "T": a.T, "warmup": a.warmup, "steps": a.steps, "reps": a.reps,
              "torch": torch.__version__, "gpus": torch.cuda.device_count(), "runs": {}}
    for B in [int(b) for b in a.batches.split(",")]:
        for prec in a.precisions.split(","):
            states = {leg: make_leg(leg, prec, B, a.T) for leg in LEGS}
            for leg in LEGS:
                run_steps(states[leg], a.warmup)
            runs = {leg: [] for leg in LEGS}
            for rep in range(a.reps):                      # legs alternate, so drifting clocks hit both alike
                for leg in LEGS:
                    r = run_steps(states[leg], a.steps)
                    runs[leg].append(r)
                    print(f"B={B} {prec} rep {rep} {leg:12s} step {r['step_ms']:8.2f} ms (wall {r['wall_step_ms']:.2f}, "
                          f"{r['hook_calls_per_step']:.0f} hook calls)", flush=True)
            med = {leg: float(np.median([r["step_ms"] for r in runs[leg]])) for leg in LEGS}
            result["runs"][f"B{B}_{prec}"] = {"step_ms_median": med, "overhead": med["passthrough"] / med["default"] - 1,
                                              "runs": runs}
            print(f"B={B} {prec}: default {med['default']:.2f} ms, passthrough {med['passthrough']:.2f} ms, overhead "
                  f"{100 * (med['passthrough'] / med['default'] - 1):+.2f} %", flush=True)
            del states
            torch.cuda.empty_cache()
    result["gpu_after"] = gpu_info()
    path = os.path.join(a.out, "sync_bn_bench.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({k: round(100 * v["overhead"], 2) for k, v in result["runs"].items()}))
    print("wrote", path)


if __name__ == "__main__":
    main()
