"""Cost of autograd through the native model beyond the plain training step, reference architecture (n_layers 12,
channels_interval 24, T = 16384), per training precision (fp32, bf16):

    train        .train(), plain input: forward + MSE loss + backward (parameter gradients) — the training step without Adam
    train_dx     .train(), x.requires_grad: the same plus the input gradient
    eval_full    .eval(), x.requires_grad, parameters requiring grad: frozen-BatchNorm forward, backward with every gradient
    eval_dx      .eval(), x.requires_grad, model.requires_grad_(False): the input-only backward of a frozen front end

Per batch size every leg runs `--warmup` untimed steps and `--steps` timed ones, and the legs alternate over `--reps`
repetitions. CUDA events around the forward (model + loss) and the backward give the per-phase device times; the medians
over the repetitions are reported. The GPU name, power limit and SM clocks are read with nvidia-smi in the same run. Writes
autograd_bench.json into --out.

    python tools/autograd_bench.py --out /tmp/agb                  # B = 64 (bench.py's per-GPU training batch)
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.train_precision_bench import gpu_info  # noqa: E402
from wave_u_net_for_speech_enhancement_b200 import Model  # noqa: E402

KINDS = ("train", "train_dx", "eval_full", "eval_dx")


def make_leg(kind, prec, B, T, seed=0):
    torch.manual_seed(seed)
    m = Model(12, 24, precision="fp32", train_precision=prec).cuda().train(kind.startswith("train"))
    if kind == "eval_dx":
        m.requires_grad_(False)
    g = torch.Generator(device="cuda").manual_seed(1)
    clean = 0.1 * torch.randn(B, 1, T, device="cuda", generator=g)
    noisy = clean + 0.05 * torch.randn(B, 1, T, device="cuda", generator=g)
    return m, noisy.requires_grad_(kind != "train"), clean


def run_steps(state, n, timed):
    m, noisy, clean = state
    crit = torch.nn.MSELoss()
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(n)]
    for i in range(n):
        m.zero_grad(set_to_none=True)
        noisy.grad = None
        e = ev[i]
        e[0].record()
        loss = crit(clean, m(noisy))                       # trainer/trainer.py:36 argument order
        e[1].record()
        loss.backward()
        e[2].record()
    torch.cuda.synchronize()
    if not timed:
        return None
    ph = np.array([[e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2])] for e in ev])
    return {"forward_ms": float(ph[:, 0].mean()), "backward_ms": float(ph[:, 1].mean()), "step_ms": float(ph.sum(1).mean())}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True, help="output directory (autograd_bench.json)")
    ap.add_argument("--batches", default="64")
    ap.add_argument("--T", type=int, default=16384)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--precisions", default="fp32,bf16")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("autograd_bench: needs a CUDA device (no CPU measurement)")
    if a.warmup < 3 or a.steps < 20 or a.reps < 3:
        sys.exit("autograd_bench: needs --warmup >= 3, --steps >= 20 and --reps >= 3")
    os.makedirs(a.out, exist_ok=True)
    legs = [(p, k) for p in a.precisions.split(",") for k in KINDS]
    result = {"gpu_before": gpu_info(), "T": a.T, "warmup": a.warmup, "steps": a.steps, "reps": a.reps,
              "torch": torch.__version__, "batches": {}}
    for B in [int(b) for b in a.batches.split(",")]:
        states = {leg: make_leg(leg[1], leg[0], B, a.T) for leg in legs}
        for leg in legs:
            run_steps(states[leg], a.warmup, timed=False)
        runs = {leg: [] for leg in legs}
        for rep in range(a.reps):                          # legs alternate, so drifting clocks hit all of them alike
            for leg in legs:
                r = run_steps(states[leg], a.steps, timed=True)
                runs[leg].append(r)
                print(f"B={B} rep {rep} {leg[0]} {leg[1]:10s} step {r['step_ms']:8.2f} ms (fwd {r['forward_ms']:.2f}, "
                      f"bwd {r['backward_ms']:.2f})", flush=True)
        summary = {}
        for leg in legs:
            med = lambda key: float(np.median([r[key] for r in runs[leg]]))  # noqa: E731
            summary[f"{leg[0]}_{leg[1]}"] = {"step_ms_median": med("step_ms"), "forward_ms": med("forward_ms"),
                                              "backward_ms": med("backward_ms"), "runs": runs[leg]}
        result["batches"][str(B)] = summary
        del states
        torch.cuda.empty_cache()
    result["gpu_after"] = gpu_info()
    path = os.path.join(a.out, "autograd_bench.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({B: {leg: (round(v["forward_ms"], 2), round(v["backward_ms"], 2)) for leg, v in s.items()}
                      for B, s in result["batches"].items()}))
    print("wrote", path)


if __name__ == "__main__":
    main()
