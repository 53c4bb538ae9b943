"""Needs a GPU: time the training trunk (forward + backward) at the BASELINE config-2 batch (256 x 3 x 256 x 128)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import ctl_b200
from ctl_b200 import synth
from ctl_b200.modelling.backbones.engine_train import TrunkTrainer

bs = int(sys.argv[1]) if len(sys.argv) > 1 else 256
sd = synth.make_trunk_state(seed=0)
params = {k: v.clone().cuda() for k, v in sd.items() if v.is_floating_point()}
tr = TrunkTrainer("cuda", graphs=os.environ.get("CTL_TRAIN_GRAPHS", "1") == "1")
x = torch.randn(bs, 3, 256, 128, device="cuda")
df = torch.randn(bs, 2048, device="cuda") * 1e-3
for w_ in range(3):
    tr.forward(x, params); torch.cuda.synchronize(); print(f"warm {w_}: forward done", flush=True)
    tr.backward(df); torch.cuda.synchronize(); print(f"warm {w_}: backward done", flush=True)
torch.cuda.synchronize()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
t0 = time.perf_counter()
it = 5
fw = bw = 0.0
for _ in range(it):
    ev[0].record(); tr.forward(x, params); ev[1].record(); g = tr.backward(df); ev[2].record()
    torch.cuda.synchronize()
    fw += ev[0].elapsed_time(ev[1]); bw += ev[1].elapsed_time(ev[2])
wall = (time.perf_counter() - t0) / it * 1e3
print(f"train trunk bs={bs}: forward {fw/it:.2f} ms, backward {bw/it:.2f} ms, wall {wall:.2f} ms/step, "
      f"{bs/((fw+bw)/it)*1e3:.0f} img/s, {3*bs*8.1065/((fw+bw)/it):.1f} TFLOP/s (3x fwd flops)")
print(f"peak memory {torch.cuda.max_memory_allocated()/2**30:.1f} GiB")
