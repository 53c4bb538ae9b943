"""Per-launch CUDA-event times of one trunk forward (needs a GPU): name, us, TFLOP/s, GB/s."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import ctl_b200
from ctl_b200.modelling.backbones.engine import TrunkEngine
from ctl_b200 import synth

bs = int(sys.argv[1]) if len(sys.argv) > 1 else 256
eng = TrunkEngine(synth.make_trunk_state(seed=0), "cuda")
x = torch.randn(bs, 3, 256, 128, device="cuda")
for _ in range(3):
    eng.forward(x)
torch.cuda.synchronize()
acc = {}
reps = 5
for _ in range(reps):
    eng.profile = []
    eng.forward(x)
    torch.cuda.synchronize()
    for i, (name, fl, by, a, b) in enumerate(eng.profile):
        k = (i, name)
        acc.setdefault(k, [0.0, fl, by])[0] += a.elapsed_time(b) * 1e3 / reps
eng.profile = None
tot = 0.0
for (i, name), (us, fl, by) in acc.items():
    tot += us
    print(f"{i:3d} {name:14s} {us:8.1f} us  {fl / us / 1e6:8.1f} TF/s  {by / us / 1e3:8.1f} GB/s")
print(f"sum {tot:.1f} us")
