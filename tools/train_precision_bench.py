"""Training-step time of the reference architecture (n_layers 12, channels_interval 24, T = 16384) in ten legs:

    native fp32   Model(train_backend="native", train_precision="fp32")   fp32 FFMA convolutions (wunet_train.cu)
    native bf16   Model(train_backend="native", train_precision="bf16")   bf16 wgmma convolutions (wunet_train_tc.cu)
    native tf32   Model(train_backend="native", train_precision="tf32")   tf32 wgmma convolutions (wunet_train_tc.cu)
    native fp16_scaled  Model(train_backend="native", train_precision="fp16_scaled")   fp16 wgmma convolutions with per-block
                  dz scaling (wunet_train_tc_f16.cu)
    *_det         the same four under torch.backends.cudnn.deterministic = True: deterministic mode (ordered weight- and
                  head-gradient sums instead of float atomics)
    autocast      Model(train_backend="torch") under torch.autocast("cuda", torch.bfloat16): PyTorch eager + cuDNN
    eager_tf32    Model(train_backend="torch") in fp32 with torch.backends.cudnn.allow_tf32 = True: PyTorch eager + cuDNN's
                  TF32 convolutions, the reference's own arithmetic on an H100

Each leg sets torch.backends.cudnn.allow_tf32 explicitly (CUDNN_TF32; True everywhere, PyTorch's default, which the legs
before eager_tf32 were measured under) and restores it afterwards.

Each step is what trainer/trainer.py:34-38 does: forward, MSE loss, backward, Adam (lr 1e-3; train.py:31-35). Per batch size
every leg runs `--warmup` untimed steps and `--steps` timed ones, and the legs alternate over `--reps` repetitions. CUDA events
around the forward (model + loss), the backward and Adam give the per-phase device times; the step time is their sum, checked
against a host clock around the whole timed window (which ends in a device synchronise). The GPU name, power limit and SM
clocks are read with nvidia-smi in the same run. Writes train_precision_bench.json into --out.

    python tools/train_precision_bench.py --out /tmp/tpb                  # B = 64 (bench.py's per-GPU batch) and 120 (train.json)
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from wave_u_net_for_speech_enhancement_b200 import Model  # noqa: E402

LEGS = {
    "native_fp32": dict(train_backend="native", train_precision="fp32"),
    "native_fp32_det": dict(train_backend="native", train_precision="fp32"),
    "native_bf16": dict(train_backend="native", train_precision="bf16"),
    "native_bf16_det": dict(train_backend="native", train_precision="bf16"),
    "native_tf32": dict(train_backend="native", train_precision="tf32"),
    "native_tf32_det": dict(train_backend="native", train_precision="tf32"),
    "native_fp16_scaled": dict(train_backend="native", train_precision="fp16_scaled"),
    "native_fp16_scaled_det": dict(train_backend="native", train_precision="fp16_scaled"),
    "autocast_bf16": dict(train_backend="torch"),
    "eager_tf32": dict(train_backend="torch"),
}
# torch.backends.cudnn.allow_tf32 per leg (only the eager legs run cuDNN convolutions; autocast's are bf16 anyway)
CUDNN_TF32 = {leg: True for leg in LEGS}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [s.strip() for s in out.splitlines()[0].split(",")]
        return {"name": name, "power_limit_w": float(power), "sm_clock_mhz": float(sm), "sm_clock_max_mhz": float(sm_max)}
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        return {"name": torch.cuda.get_device_name(), "nvidia_smi_error": repr(e)}


def make_leg(leg, B, T, seed=0):
    torch.manual_seed(seed)
    m = Model(12, 24, precision="fp32", **LEGS[leg]).cuda().train()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, betas=(0.9, 0.999))
    g = torch.Generator(device="cuda").manual_seed(1)
    clean = 0.1 * torch.randn(B, 1, T, device="cuda", generator=g)
    noisy = clean + 0.05 * torch.randn(B, 1, T, device="cuda", generator=g)
    return m, opt, noisy, clean


def run_steps(leg, state, n, timed):
    m, opt, noisy, clean = state
    autocast = leg == "autocast_bf16"
    crit = torch.nn.MSELoss()
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(n)]
    losses = []
    saved = torch.backends.cudnn.deterministic, torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.deterministic = leg.endswith("_det")
    torch.backends.cudnn.allow_tf32 = CUDNN_TF32[leg]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(n):
        e = ev[i]
        e[0].record()
        opt.zero_grad()
        with torch.autocast("cuda", torch.bfloat16, enabled=autocast):
            y = m(noisy)
            loss = crit(clean, y.float())                  # trainer/trainer.py:36 argument order
        e[1].record()
        loss.backward()
        e[2].record()
        opt.step()
        e[3].record()
        losses.append(loss.detach())
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    torch.backends.cudnn.deterministic, torch.backends.cudnn.allow_tf32 = saved
    if not timed:
        return None
    ph = np.array([[e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]), e[2].elapsed_time(e[3])] for e in ev])
    return {"forward_ms": float(ph[:, 0].mean()), "backward_ms": float(ph[:, 1].mean()), "adam_ms": float(ph[:, 2].mean()),
            "step_ms": float(ph.sum(1).mean()), "wall_step_ms": 1e3 * wall / n,
            "first_loss": float(losses[0]), "last_loss": float(losses[-1])}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True, help="output directory (train_precision_bench.json)")
    ap.add_argument("--batches", default="64,120")
    ap.add_argument("--T", type=int, default=16384)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--legs", default=",".join(LEGS))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_precision_bench: needs a CUDA device (no CPU measurement)")
    if a.warmup < 3 or a.steps < 20 or a.reps < 3:
        sys.exit("train_precision_bench: needs --warmup >= 3, --steps >= 20 and --reps >= 3")
    os.makedirs(a.out, exist_ok=True)
    legs = a.legs.split(",")
    result = {"gpu_before": gpu_info(), "T": a.T, "warmup": a.warmup, "steps": a.steps, "reps": a.reps,
              "torch": torch.__version__, "cudnn": torch.backends.cudnn.version(),
              "cudnn_allow_tf32": {leg: CUDNN_TF32[leg] for leg in legs}, "batches": {}}
    for B in [int(b) for b in a.batches.split(",")]:
        states = {leg: make_leg(leg, B, a.T) for leg in legs}
        for leg in legs:
            run_steps(leg, states[leg], a.warmup, timed=False)
        runs = {leg: [] for leg in legs}
        for rep in range(a.reps):                          # legs alternate, so drifting clocks hit all of them alike
            for leg in legs:
                r = run_steps(leg, states[leg], a.steps, timed=True)
                runs[leg].append(r)
                print(f"B={B} rep {rep} {leg:22s} step {r['step_ms']:8.2f} ms (fwd {r['forward_ms']:.2f}, bwd {r['backward_ms']:.2f}, "
                      f"adam {r['adam_ms']:.2f}; wall {r['wall_step_ms']:.2f})", flush=True)
        summary = {}
        for leg in legs:
            st = np.array([r["step_ms"] for r in runs[leg]])
            summary[leg] = {"step_ms_median": float(np.median(st)), "step_ms_min": float(st.min()), "step_ms_max": float(st.max()),
                            "frames_per_s": float(B / (np.median(st) * 1e-3)),
                            "forward_ms": float(np.median([r["forward_ms"] for r in runs[leg]])),
                            "backward_ms": float(np.median([r["backward_ms"] for r in runs[leg]])),
                            "adam_ms": float(np.median([r["adam_ms"] for r in runs[leg]])), "runs": runs[leg]}
        result["batches"][str(B)] = summary
        del states
        torch.cuda.empty_cache()
    result["gpu_after"] = gpu_info()
    path = os.path.join(a.out, "train_precision_bench.json")
    with open(path, "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({B: {leg: round(v["step_ms_median"], 2) for leg, v in s.items()} for B, s in result["batches"].items()}))
    print("wrote", path)


if __name__ == "__main__":
    main()
