"""Development check of the bf16 tensor-core path: per-level max error vs the golden vectors (GPU box)."""
import os, sys
os.environ.setdefault("WUNET_TC_STORE_LAST", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model

def run(n, ci, st, x, levels_ref=None, y_ref=None, tag=""):
    m = Model(n, ci, precision="bf16")
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()})
    m = m.to("cuda:0").eval()
    with torch.no_grad():
        y = m(torch.from_numpy(x).cuda())
    torch.cuda.synchronize()
    y = y.cpu().numpy()
    B, _, T = x.shape
    worst = 0.0
    for i in range(2 * n + 1):
        lv = m.read_level(i, B, T).cpu().numpy()
        ref = levels_ref[i]
        err = np.abs(lv - ref).max(); scale = np.abs(ref).max()
        worst = max(worst, err / scale)
        print(f"{tag} level {i:2d} shape {lv.shape} max_err {err:.4e} ref_max {scale:.3f} rel {err/scale:.4f}", flush=True)
    print(f"{tag} output max_err {np.abs(y - y_ref).max():.4e}  (max|y| {np.abs(y_ref).max():.3f})", flush=True)
    return worst

if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    if which in ("small", "all"):
        g = np.load(os.path.join(ROOT, "tests/golden/small_n4_c8.npz"))
        n, ci, T, B = 4, 8, 256, 3
        st = wo.make_state(n, ci, seed=11); x = wo.make_input(B, T, seed=12)
        run(n, ci, st, x, [g[f"level_{i}"] for i in range(2 * n + 1)], g["y"], "small")
    if which in ("full", "all"):
        n, ci, T, B = 12, 24, 16384, 2
        st = wo.make_state(n, ci, seed=0); x = wo.make_input(B, T, seed=1234)
        y, levels = wo.COracle(n, ci).forward(st, x, return_levels=True)
        run(n, ci, st, x, levels, y, "full")
    if which in ("b5", "all"):
        n, ci, T, B = 12, 24, 4096, 5
        st = wo.make_state(n, ci, seed=0); x = wo.make_input(B, T, seed=77)
        y, levels = wo.COracle(n, ci).forward(st, x, return_levels=True)
        run(n, ci, st, x, levels, y, "T4096_B5")
