"""One configuration of the row-pair experiment (WUNET_TC_PAIR) on the GPU: correctness against the C oracle and the default
path, per-block outputs of the two blocks it changes, and per-block times at batch 256. One process per configuration, so
that a hang in an experimental kernel is contained by `timeout`:

    timeout 120 python tools/pair_check.py <pair mask 0..1> [WUNET_TC_OVR string]

Prints one JSON line (also appended to gpurun_out/pair/results.jsonl)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
MASK = sys.argv[1] if len(sys.argv) > 1 else "0"
OVR = sys.argv[2] if len(sys.argv) > 2 else ""
os.environ["WUNET_TC_PAIR"] = MASK
os.environ["WUNET_TC_STORE_LAST"] = "1"            # small-batch leg: also materialise the last block (per-block comparison)
if OVR:
    os.environ["WUNET_TC_OVR"] = OVR

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import wunet_oracle as wo  # noqa: E402  (checker only)
from wave_u_net_for_speech_enhancement_b200 import Model  # noqa: E402

n, ci, T = 12, 24, 16384
st = wo.make_state(n, ci, seed=0)
sd = {k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}
res = {"pair": int(MASK), "ovr": OVR, "enc0_tc": os.environ.get("WUNET_TC_ENC0", "0")}


def make():
    m = Model(n, ci, precision="bf16")
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


# ---- small batch: output and the two affected blocks against the oracle (fp64-accumulated C restatement of the reference)
B = 2
x = wo.make_input(B, T, seed=1234)
# edge vectors in frame 1: impulses at the first and last sample on top of the noise (conv zero padding, upsample end points)
x[1, 0, 0] += 0.9
x[1, 0, T - 1] -= 0.9
want, olv = wo.COracle(n, ci).forward(st, x, return_levels=True)
os.makedirs(os.path.join(ROOT, "gpurun_out", "pair"), exist_ok=True)
m = make()
with torch.no_grad():
    y = m(torch.from_numpy(x).cuda())
torch.cuda.synchronize()
yh = y.cpu().numpy()
err = np.abs(yh - want)
res["finite"] = bool(np.isfinite(yh).all())
res["out_err_max"] = float(err.max())
res["out_err_even"] = float(err[..., 0::2].max())
res["out_err_odd"] = float(err[..., 1::2].max())
res["out_err_first8"] = [round(float(v), 5) for v in err[1, 0, :8]]
res["out_err_last8"] = [round(float(v), 5) for v in err[1, 0, -8:]]
res["out_err_argmax"] = [int(v) for v in np.unravel_index(int(err.argmax()), err.shape)]
blk = {}
for b in (0, 1, 2, 2 * n - 1, 2 * n):
    a = m.read_level(b, B, T).cpu().numpy()
    blk[b] = a
    res[f"blk{b}_absmax"] = float(np.abs(a).max())
    # relative error of the block against the oracle's fp32 activations (bf16 operands: ~0.3-0.5 % of the block's max)
    res[f"blk{b}_rel_vs_oracle"] = float(np.abs(a - olv[b]).max() / np.abs(olv[b]).max())
# the default path's blocks, for a direct A/B of the blocks themselves (bf16 rounding of the same arithmetic)
ref_file = os.path.join(ROOT, "gpurun_out", "pair", "blk_ref.npz")
if MASK in ("0", "1") and not OVR and os.environ.get("WUNET_TC_ENC0", "0") != "1" and not os.path.exists(ref_file):
    np.savez(ref_file, **{f"b{k}": v for k, v in blk.items()}, y=yh)
elif os.path.exists(ref_file):
    ref = np.load(ref_file)
    for b in (0, 1, 2 * n):
        d = np.abs(blk[b] - ref[f"b{b}"])
        scale = float(np.abs(ref[f"b{b}"]).max())
        res[f"blk{b}_vs_default_max"] = float(d.max())
        res[f"blk{b}_vs_default_rel"] = float(d.max() / scale)
        res[f"blk{b}_vs_default_mean"] = float(d.mean())
        # where is the worst element: (frame, channel, position) - a layout bug shows as a pattern, rounding noise does not
        res[f"blk{b}_argmax"] = [int(v) for v in np.unravel_index(int(d.argmax()), d.shape)]
        res[f"blk{b}_err_by_parity"] = [float(d[..., 0::2].max()), float(d[..., 1::2].max())]
        res[f"blk{b}_err_by_chan8"] = [round(float(d[:, c:c + 8].max()), 4) for c in range(0, d.shape[1], 8)]
        res[f"blk{b}_err_edges"] = [round(float(d[..., :4].max()), 4), round(float(d[..., -4:].max()), 4)]
    res["y_vs_default_max"] = float(np.abs(yh - ref["y"]).max())
m._release()
del m

# ---- batch 256, the benchmarked variant (no store of the last block): times per block, and 16 frames against the oracle
os.environ["WUNET_TC_STORE_LAST"] = "0"
B = 256
xb = wo.make_input(B, T, seed=77)
m = make()
xt = torch.from_numpy(xb).cuda()
with torch.no_grad():
    y = m(xt)
    torch.cuda.synchronize()
    m.profile(True)
    tot = None
    reps = 10
    for _ in range(reps):
        y = m(xt)
        ms = np.array(m.profile_read())
        tot = ms if tot is None else tot + ms
    m.profile(False)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        m(xt)
    e0.record()
    for _ in range(20):
        m(xt)
    e1.record()
    torch.cuda.synchronize()
tot = tot / reps
idx = list(range(0, B, 32))
want = wo.COracle(n, ci).forward(st, xb[idx])
res["b256_err_8frames"] = float(np.abs(y.cpu().numpy()[idx] - want).max())
res["b256_step_ms"] = round(e0.elapsed_time(e1) / 20, 4)
res["b256_sum_blocks_ms"] = round(float(tot.sum()), 4)
res["b256_blocks_us"] = [round(float(v) * 1e3, 1) for v in tot[:2 * n + 1]]
res["launches"] = m.last_launch_count()
m._release()
line = json.dumps(res)
print(line, flush=True)
os.makedirs(os.path.join(ROOT, "gpurun_out", "pair"), exist_ok=True)
with open(os.path.join(ROOT, "gpurun_out", "pair", "results.jsonl"), "a") as f:
    f.write(line + "\n")
