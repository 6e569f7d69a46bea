"""Per-role clock64 timelines of CTA 0 for the given blocks (needs a WUNET_TC_TRACE build of the library, see build.py):

    WUNET_TC_TRACE=1 python -m wave_u_net_for_speech_enhancement_b200.build --force   # then move the .so aside
    WUNET_LIB_PATH=.../libwunet_b200_trace.so python tools/trace_levels.py 23 22 2> trace.txt

Roles: 0 = TMA producer (around its operand-stage waits, after each weight-stage wait), 1 = consumer thread 0 (before / after
each operand-stage wait), 2 = consumer thread 0 at the start of each epilogue, 4 = upsample producer thread 0 (before / after
the stage wait, after the hand-off). Times are clock64 cycles from role 1's first stamp.
Blocks that run the ping-pong form (wunet_tc_pp.cuh) stamp per tile of each consumer warpgroup, role 1 for warpgroup 0 (thread
0) and role 3 for warpgroup 1 (thread 128): MMA turn taken, MMAs done (= epilogue start), epilogue done; role 2 stays empty.
Blocks that run in 256-row units (wunet_tc_m2.cuh) stamp role 1 before / after each weight-stage wait instead of each
operand-stage wait; role 2 is the start of each unit's epilogue.
"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
from oracle import wunet_oracle as wo
from wave_u_net_for_speech_enhancement_b200 import Model

st = wo.make_state(12, 24, seed=0)
sd = {k: torch.from_numpy(np.asarray(v)) for k, v in st.items()}
x = torch.from_numpy(wo.make_input(256, 16384, seed=1)).cuda()
for lvl in sys.argv[1:]:
    os.environ["WUNET_TC_TRACE_LEVEL"] = lvl
    os.environ["WUNET_TC_DEBUG"] = "1" if lvl == sys.argv[1] else ""
    if not os.environ["WUNET_TC_DEBUG"]:
        os.environ.pop("WUNET_TC_DEBUG")
    m = Model(12, 24, precision="bf16")
    m.load_state_dict(sd)
    m = m.cuda().eval()
    with torch.no_grad():
        for _ in range(2):
            m(x)
    torch.cuda.synchronize()
    sys.stderr.write("[trace block %s]\n" % lvl)
    sys.stderr.flush()
    m._release()
