"""Time the fused stem (pack + conv/pool kernels) alone (needs a GPU)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from ctl_b200 import _native as N
from ctl_b200.modelling.backbones.engine import pack_stem_fused
L = N.lib()
n, H, W = 256, 256, 128
xs = [torch.randn(n, 3, H, W, device="cuda") for _ in range(3)]
w = pack_stem_fused(torch.randn(64, 3, 7, 7, device="cuda") * 0.1)
b = torch.randn(64, device="cuda")
pad = torch.zeros(L.ctl_stem_pad_bytes(n, H, W), dtype=torch.uint8, device="cuda")
out = torch.empty(n, H // 4, W // 4, 64, dtype=torch.float16, device="cuda")
def run(i):
    N.check(L.ctl_stem_pool_fused(xs[i % 3].data_ptr(), n, H, W, pad.data_ptr(), w.data_ptr(), b.data_ptr(), 0, out.data_ptr(), N.stream_ptr()))
for i in range(5): run(i)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for i in range(20): run(i)
e1.record(); torch.cuda.synchronize()
print(f"pack+stem_pool {e0.elapsed_time(e1)/20*1e3:.1f} us")
