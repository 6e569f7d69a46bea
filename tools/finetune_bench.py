"""Fine-tuning step time of the native training step: forward and backward ms per step at B = 64 and 120, T = 16384, fp32 and
bf16, in four configurations, legs alternated round by round on one model:

  full          every BatchNorm in training mode, every parameter trainable;
  bn_frozen     every BatchNorm container in .eval() (running statistics), every parameter trainable;
  enc_mid       encoder + middle frozen: their BatchNorm in .eval() and requires_grad_(False);
  head_only     every BatchNorm in .eval(), only the 1x1 output conv trainable.

Loss = MSELoss(clean, y) as in the reference trainer; the forward is timed from the call to y, the backward over
loss.backward(), each with CUDA events and a synchronise. Writes the table and the GPU's name, power limit and SM clock to
--out (JSON) and prints it.

    python tools/finetune_bench.py --out /tmp/finetune.json
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wave_u_net_for_speech_enhancement_b200 import Model  # noqa: E402

CONFIGS = ["full", "bn_frozen", "enc_mid", "head_only"]


def configure(m, cfg):
    m.train()
    m.requires_grad_(True)
    bns = [blk[1] for blk in m._blocks()]
    if cfg in ("bn_frozen", "head_only"):
        for bn in bns:
            bn.eval()
    if cfg == "enc_mid":
        for bn in bns[:m.n_layers + 1]:
            bn.eval()
        m.encoder.requires_grad_(False)
        m.middle.requires_grad_(False)
    if cfg == "head_only":
        m.requires_grad_(False)
        m.out.requires_grad_(True)


def timed_steps(m, x, clean, steps):
    fwd = bwd = 0.0
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    for _ in range(steps):
        m.zero_grad(set_to_none=True)
        ev[0].record()
        y = m(x)
        ev[1].record()
        torch.nn.MSELoss()(clean, y).backward()
        ev[2].record()
        torch.cuda.synchronize()
        fwd += ev[0].elapsed_time(ev[1])
        bwd += ev[1].elapsed_time(ev[2])
    return fwd, bwd


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="64,120")
    ap.add_argument("--T", type=int, default=16384)
    ap.add_argument("--precisions", default="fp32,bf16")
    ap.add_argument("--steps", type=int, default=5, help="timed steps per leg and round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("finetune_bench needs a CUDA device")
    info = gpu_info()
    rows = []
    for prec in a.precisions.split(","):
        torch.manual_seed(0)
        m = Model(train_precision=prec).cuda()
        for B in (int(b) for b in a.batches.split(",")):
            g = torch.Generator(device="cuda").manual_seed(1)
            clean = 0.1 * torch.randn(B, 1, a.T, device="cuda", generator=g)
            x = clean + 0.05 * torch.randn(B, 1, a.T, device="cuda", generator=g)
            tot = {c: [0.0, 0.0, 0] for c in CONFIGS}
            for cfg in CONFIGS:
                configure(m, cfg)
                timed_steps(m, x, clean, a.warmup)
            for _ in range(a.rounds):
                for cfg in CONFIGS:
                    configure(m, cfg)
                    f, b = timed_steps(m, x, clean, a.steps)
                    tot[cfg][0] += f
                    tot[cfg][1] += b
                    tot[cfg][2] += a.steps
            for cfg in CONFIGS:
                f, b, k = tot[cfg]
                rows.append({"precision": prec, "B": B, "T": a.T, "config": cfg, "forward_ms": f / k, "backward_ms": b / k,
                             "step_ms": (f + b) / k, "steps": k})
                print(f"{prec:5s} B={B:4d} {cfg:10s} forward {f / k:8.2f} ms  backward {b / k:8.2f} ms  step {(f + b) / k:8.2f} ms",
                      flush=True)
        del m
        torch.cuda.empty_cache()
    res = {"gpu": info, "rows": rows}
    print(json.dumps(info))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
