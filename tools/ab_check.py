"""A/B of a kernel-path switch of the bf16 path (environment variable read when the library creates a context, "0" = off):
output difference and per-block times, plus the error of both against the fp32 path on a few frames.

    timeout 120 python tools/ab_check.py WUNET_TC_GEMM      # dense GEMM over frames for the blocks of <= 16 samples
    timeout 120 python tools/ab_check.py WUNET_TC_MERGE     # merged decoder tail chunk
    timeout 120 python tools/ab_check.py WUNET_TC_M2        # 256-row units for the streamed-weight blocks
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from wave_u_net_for_speech_enhancement_b200 import Model  # noqa: E402


VAR = sys.argv[1] if len(sys.argv) > 1 else "WUNET_TC_GEMM"


def run(on, B, reps=5, precision="bf16"):
    os.environ[VAR] = "1" if on else "0"                      # read when the library creates the model's tensor-core state
    torch.manual_seed(0)
    m = Model(12, 24, precision=precision).cuda().eval()
    with torch.no_grad():                                     # eval-BatchNorm far from identity, like the parity tests
        g = torch.Generator().manual_seed(7)
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm1d):
                mod.running_mean.copy_(0.1 * torch.randn(mod.running_mean.shape, generator=g))
                mod.running_var.copy_(0.5 + torch.rand(mod.running_var.shape, generator=g))
                mod.weight.copy_(0.5 + torch.rand(mod.weight.shape, generator=g))
                mod.bias.copy_(0.1 * torch.randn(mod.bias.shape, generator=g))
    x = 0.3 * torch.randn(B, 1, 16384, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    with torch.no_grad():
        y = m(x)
        m.profile(True)
        tot = None
        for _ in range(reps):
            y = m(x)
            ms = np.array(m.profile_read())
            tot = ms if tot is None else tot + ms
    torch.cuda.synchronize()
    y = y.clone()
    m._release()
    return y, tot / reps


for B in (3, 256):
    y0, t0 = run(False, B)
    y1, t1 = run(True, B)
    print("B=%d: %s off %.4f ms, on %.4f ms, max|on - off| %.3e, finite %s" % (B, VAR, t0.sum(), t1.sum(), float((y1 - y0).abs().max()),
                                                                               bool(torch.isfinite(y1).all())), flush=True)
    if B == 3:
        y32, _ = run(True, B, reps=1, precision="fp32")
        print("   vs the fp32 path: off %.3e, on %.3e" % (float((y0 - y32).abs().max()), float((y1 - y32).abs().max())), flush=True)
    if B == 256:
        print("   per block us: " + " ".join("%d:%.0f>%.0f" % (i, a * 1e3, b * 1e3) for i, (a, b) in enumerate(zip(t0, t1)) if i < 25))
