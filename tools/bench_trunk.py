"""Quick device-side timing of the trunk engine (needs a GPU)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import ctl_b200
from ctl_b200.modelling.backbones.engine import TrunkEngine
from ctl_b200 import synth

bs = int(sys.argv[1]) if len(sys.argv) > 1 else 256
sd = synth.make_trunk_state(seed=0)
eng = TrunkEngine(sd, "cuda")
x = torch.randn(bs, 3, 256, 128, device="cuda")
for _ in range(3):
    eng.forward(x)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
iters = 10
for _ in range(iters):
    eng.forward(x)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / iters
print(f"trunk fwd bs={bs}: {ms:.3f} ms -> {bs/ms*1e3:.0f} img/s, {bs*8.1065/ms:.1f} TFLOP/s")
if os.environ.get("CTL_GRAPH", "1") == "1":
    from ctl_b200.modelling.backbones.engine import GraphedForward
    gf = GraphedForward(eng, x, want_emb=False)
    for _ in range(3):
        gf()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        gf()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    print(f"trunk fwd bs={bs} (CUDA graph): {ms:.3f} ms -> {bs/ms*1e3:.0f} img/s, {bs*8.1065/ms:.1f} TFLOP/s")
