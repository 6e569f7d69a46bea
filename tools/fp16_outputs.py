"""Save the fp16 forward's output at the benchmark shape (12 levels x 24 base filters, batch 256 x 16384 samples, seeded state and
input) as y.npy, so that two builds can be compared byte for byte:

    python tools/fp16_outputs.py OUT_DIR [--root TREE]

--root: the repository tree whose package runs (default: this one), e.g. a checkout of another commit with its library built.
"""
import argparse
import os
import sys

ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
ap.add_argument("out")
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--batch", type=int, default=256)
a = ap.parse_args()
sys.path.insert(0, os.path.abspath(a.root))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from oracle import wunet_oracle as wo  # noqa: E402
from wave_u_net_for_speech_enhancement_b200 import Model  # noqa: E402

st = wo.make_state(12, 24, seed=0)
m = Model(12, 24, precision="fp16")
m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}, strict=True)
m = m.cuda().eval()
x = torch.from_numpy(wo.make_input(a.batch, 16384, seed=1)).cuda()
with torch.no_grad():
    y = m(x)
torch.cuda.synchronize()
os.makedirs(a.out, exist_ok=True)
np.save(os.path.join(a.out, "y.npy"), y.cpu().numpy())
print("saved", os.path.join(a.out, "y.npy"), "from", os.path.abspath(a.root), tuple(y.shape))
m._release()
