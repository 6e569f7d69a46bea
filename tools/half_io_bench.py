"""float32 I/O against fp16 I/O at precision="bf16", B x T = 256 x 16384: the same weights (fp16 values) in a float32 model and
in its .half() copy, legs alternated. Two measurements:
  device   the device-resident forward (CUDA events around `iters` calls; input and output on the GPU);
  stream   end to end through forward_host_stream with pinned host buffers (host clock around `batches` batches, which ends
           when the last output is on the host).
Prints one JSON line with the card's name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import wunet_oracle as wo  # noqa: E402
from wave_u_net_for_speech_enhancement_b200 import Model  # noqa: E402


def device_ms(m, x, iters):
    with torch.no_grad():
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(iters):
            m(x)
        end.record()
        torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def stream_ms(m, xs, outs):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in m.forward_host_stream(xs, outs):
        pass
    return (time.perf_counter() - t0) * 1e3 / len(xs)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--B", type=int, default=256)
    ap.add_argument("--T", type=int, default=16384)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--batches", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("half_io_bench needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    sd = {k: torch.from_numpy(v).half().float() if v.dtype.kind == "f" else torch.from_numpy(v)
          for k, v in wo.make_state(12, 24, seed=0).items()}
    legs = {}
    for name, dtype in (("f32_io", torch.float32), ("f16_io", torch.float16)):
        m = Model(12, 24, precision="bf16")
        m.load_state_dict(sd, strict=True)
        m = m.cuda().to(dtype).eval()
        x = torch.from_numpy(wo.make_input(a.B, a.T)).to(dtype)
        xs = [x.clone().pin_memory() for _ in range(a.batches)]
        outs = [torch.empty_like(x).pin_memory() for _ in range(a.batches)]
        legs[name] = (m, x.cuda(), xs, outs)
        device_ms(m, legs[name][1], 5)                              # warm-up: plan, packing, module load
        stream_ms(m, xs[:4], outs[:4])
    res = {k: {"device_ms": [], "stream_ms_per_batch": []} for k in legs}
    for _ in range(a.rounds):
        for k, (m, xd, xs, outs) in legs.items():
            res[k]["device_ms"].append(round(device_ms(m, xd, a.iters), 4))
            res[k]["stream_ms_per_batch"].append(round(stream_ms(m, xs, outs), 3))
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    print(json.dumps({"gpu": smi, "B": a.B, "T": a.T, "precision": "bf16", "legs": res,
                      "median": {k: {kk: med(vv) for kk, vv in v.items()} for k, v in res.items()}}))


if __name__ == "__main__":
    main()
