"""Needs a GPU: topk_and_eval at a config-5 shard shape (16384 x 25000 x 2048) -- caller order vs identity order + tile lists."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import ctl_b200  # noqa: F401
from ctl_b200 import retrieval as R

NQ, NG, D, IDS = 16384, 25000, 2048, 4000
g = torch.Generator(device="cuda").manual_seed(3)
cent = torch.randn(IDS, D, device="cuda", generator=g)
pid = torch.randint(0, IDS, (NQ + NG,), device="cuda", generator=g)
cam = torch.randint(0, 6, (NQ + NG,), device="cuda", generator=g)
f = torch.nn.functional.normalize(cent[pid] + 3.0 * torch.randn(NQ + NG, D, device="cuda", generator=g), dim=1)
pids, cams = pid.cpu().numpy(), cam.cpu().numpy()
q, gal = f[:NQ].contiguous(), f[NQ:].contiguous()
args = (pids[:NQ], pids[NQ:], cams[:NQ], cams[NQ:])
qo, go = R.pid_order(pids[:NQ]), R.pid_order(pids[NQ:])
ids_u = R.encode_ids(*args, False, q.device)
ids_s = R.encode_ids(*args, False, q.device, q_order=qo, g_order=go)
cache = R.PlaneCache()


def T(fn, n=5):
    fn(); torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n): fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e3


a = R.topk_and_eval(R.build_planes(q), cache.get(gal), 100, *args, ids=ids_u)
b = R.topk_and_eval(R.build_planes(q, order=qo), cache.get(gal, order=go), 100, *args, ids=ids_s)
print("identical:", bool(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2].mAP == b[2].mAP), "mAP", a[2].mAP)
print("caller order               %.3f ms" % T(lambda: R.topk_and_eval(R.build_planes(q), cache.get(gal), 100, *args, ids=ids_u)))
print("pid order, every tile      %.3f ms" % T(lambda: R.topk_and_eval(R.build_planes(q, order=qo), cache.get(gal, order=go), 100, *args, ids=ids_s, tile_lists=False)))
print("pid order, tile lists      %.3f ms" % T(lambda: R.topk_and_eval(R.build_planes(q, order=qo), cache.get(gal, order=go), 100, *args, ids=ids_s)))
print("evaluate_streamed caller   %.3f ms" % T(lambda: R.evaluate_streamed(R.build_planes(q), cache.get(gal), *args, ids=ids_u)))
print("evaluate_streamed pid ord. %.3f ms" % T(lambda: R.evaluate_streamed(R.build_planes(q, order=qo), cache.get(gal, order=go), *args, ids=ids_s)))
