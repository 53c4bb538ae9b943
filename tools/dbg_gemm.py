"""Debug helper (needs a GPU): distance matrix of tiny / structured inputs vs torch, with a
pattern dump when something is off."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import ctl_b200
from ctl_b200 import retrieval as R

torch.manual_seed(0)
for (nq, ng, d) in [(128, 128, 64), (128, 128, 128), (128, 256, 2048), (200, 300, 2048), (3368, 15913, 2048)]:
    q = torch.randn(nq, d, device="cuda")
    g = torch.randn(ng, d, device="cuda")
    out = R.dist_matrix(q, g)
    torch.cuda.synchronize()
    ref = (q.double() ** 2).sum(1)[:, None] + (g.double() ** 2).sum(1)[None, :] - 2 * q.double() @ g.double().t()
    err = (out.double() - ref).abs()
    scale = float(ref.abs().max())
    print(f"nq={nq} ng={ng} d={d}: max abs err {float(err.max()):.3e} (scale {scale:.1f}) rel {float(err.max())/scale:.2e}")
    if float(err.max()) / scale > 1e-5:
        bad = (err / scale > 1e-5)
        print("  bad fraction", float(bad.float().mean()))
        print("  bad rows (first 16):", bad.any(1).nonzero().flatten()[:16].tolist())
        print("  bad cols (first 16):", bad.any(0).nonzero().flatten()[:16].tolist())
        print("  out[0,:8]", out[0, :8].tolist())
        print("  ref[0,:8]", ref[0, :8].tolist())
        # structured probe: one-hot rows reveal k / row permutations
        qe = torch.zeros(nq, d, device="cuda"); ge = torch.zeros(ng, d, device="cuda")
        qe[torch.arange(nq), torch.arange(nq) % d] = 1.0
        ge[torch.arange(ng), torch.arange(ng) % d] = 1.0
        oe = R.dist_matrix(qe, ge)
        dot = (2.0 - oe) / 2.0
        print("  one-hot probe: dot[0,:16]", dot[0, :16].tolist())
        print("  one-hot probe: dot[:16,0]", dot[:16, 0].tolist())
        print("  one-hot probe: argmax col per row (first 16)", dot[:16].argmax(1).tolist())
        break
import time
q = torch.randn(3368, 2048, device="cuda"); g = torch.randn(15913, 2048, device="cuda")
qp, gp = R.build_planes(q), R.build_planes(g)
for _ in range(2):
    idx, dst, ovf = R.topk(qp, gp, 100)
torch.cuda.synchronize()
t0 = time.time()
for _ in range(5):
    idx, dst, ovf = R.topk(qp, gp, 100)
torch.cuda.synchronize()
dt = (time.time() - t0) / 5
print(f"topk 3368x15913 k=100: {dt*1e3:.3f} ms -> {3368*15913/dt/1e9:.2f} Gpairs/s, ovf={int(ovf)}")
