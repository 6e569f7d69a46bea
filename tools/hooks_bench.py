"""Cost of forward hooks on the block containers (H100): the bf16 eval forward at B = 256 x 16384 with no hook, one hook on
decoder[n-1] and a hook on each of the 2n+2 top-level containers (encoder[i], middle, decoder[j], out), and the native bf16
training step at B = 64 with and without a feature loss on four decoder levels. Legs alternate round by round; each number is
the median over rounds of the mean step time of one round (CUDA events). Prints one JSON line, with the card, its power limit
and SM clock read in the same run.

    python tools/hooks_bench.py [--rounds 5] [--steps 20]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import wunet_oracle as wo  # noqa: E402
from wave_u_net_for_speech_enhancement_b200 import Model  # noqa: E402

N, CI, T = 12, 24, 16384


def timed(fn, steps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    st = {k: torch.from_numpy(v) for k, v in wo.make_state(N, CI, seed=0).items()}
    dev = "cuda:0"

    m = Model(N, CI, precision="bf16")
    m.load_state_dict(st)
    m = m.to(dev).eval()
    x = torch.from_numpy(wo.make_input(256, T, seed=1)).to(dev)
    sink = []

    def fwd():
        with torch.no_grad():
            m(x)
        sink.clear()

    def hook(mod, args, out):
        sink.append(out)

    tops = list(m.encoder) + [m.middle] + list(m.decoder) + [m.out]
    legs = {"forward_no_hook": [], "forward_hook_last_decoder": [], "forward_hook_all_2n+2": []}
    for _ in range(a.rounds):
        legs["forward_no_hook"].append(timed(fwd, a.steps))
        h = m.decoder[N - 1].register_forward_hook(hook)
        legs["forward_hook_last_decoder"].append(timed(fwd, a.steps))
        h.remove()
        hs = [t.register_forward_hook(hook) for t in tops]
        legs["forward_hook_all_2n+2"].append(timed(fwd, a.steps))
        for h in hs:
            h.remove()
    del m, x

    tm = Model(N, CI, train_precision="bf16")
    tm.load_state_dict(st)
    tm = tm.to(dev).train()
    opt = torch.optim.Adam(tm.parameters(), lr=1e-6)
    g = torch.Generator(device=dev).manual_seed(2)
    noisy = torch.randn(64, 1, T, device=dev, generator=g) * 0.1
    clean = torch.randn(64, 1, T, device=dev, generator=g) * 0.1
    feats = {}
    dec = [N - 4, N - 3, N - 2, N - 1]

    def train_step(feature):
        hs = [tm.decoder[j].register_forward_hook(lambda mod, a, o, j=j: feats.__setitem__(j, o)) for j in dec] if feature else []
        y = tm(noisy)
        loss = F.mse_loss(y, clean)
        for j in dec if feature else []:
            loss = loss + 0.1 * feats[j].pow(2).mean()
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        for h in hs:
            h.remove()
        feats.clear()

    legs.update({"train_no_feature_loss": [], "train_feature_loss_4_decoders": []})
    for _ in range(a.rounds):
        legs["train_no_feature_loss"].append(timed(lambda: train_step(False), a.steps // 2))
        legs["train_feature_loss_4_decoders"].append(timed(lambda: train_step(True), a.steps // 2))

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    out = {k + "_ms": round(statistics.median(v), 3) for k, v in legs.items()}
    out.update({"spread_ms": {k: round(max(v) - min(v), 3) for k, v in legs.items()}, "gpu": q, "rounds": a.rounds,
                "steps": a.steps, "forward_batch": 256, "train_batch": 64, "T": T})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
