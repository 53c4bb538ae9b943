"""Needs a GPU: where one retrieval step (top-100 + CMC/mAP) spends its time -- host enqueue vs device for every variant
(caller order, identity order, tile lists, top-k only, evaluation only), the passes alone, the candidate volume of the
two thresholds.  --shape config3: 3368 x 15913 x 2048 (Market-like, synth.synth_retrieval); shard5: one rank's share of
config 5, 16384 x 25000 x 2048 (4000 identities, unit-norm rows generated on the device).  Prints the card's name and
power limit."""
import argparse
import ctypes as C
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import ctl_b200  # noqa: F401
from ctl_b200 import _native as N
from ctl_b200 import retrieval as R
from ctl_b200 import synth
from tools.bench_basic import card

ap = argparse.ArgumentParser()
ap.add_argument("--shape", default="config3", choices=["config3", "shard5"])
SHAPE = ap.parse_args().shape
if SHAPE == "config3":
    NQ, NG, D = 3368, 15913, 2048
    feats, pids, cams = synth.synth_retrieval(NQ, NG, 751, D, 3.0, 0)
    q, g = feats[:NQ].cuda(), feats[NQ:].cuda()
else:
    NQ, NG, D, IDS = 16384, 25000, 2048, 4000
    gen = torch.Generator(device="cuda").manual_seed(3)
    cent = torch.randn(IDS, D, device="cuda", generator=gen)
    pid = torch.randint(0, IDS, (NQ + NG,), device="cuda", generator=gen)
    cam = torch.randint(0, 6, (NQ + NG,), device="cuda", generator=gen)
    f = torch.nn.functional.normalize(cent[pid] + 3.0 * torch.randn(NQ + NG, D, device="cuda", generator=gen), dim=1)
    pids, cams = pid.cpu().numpy(), cam.cpu().numpy()
    q, g = f[:NQ].contiguous(), f[NQ:].contiguous()
name, power = card()
print(f"{SHAPE}: {NQ} x {NG} x {D} on {name} at a {power} power limit")
qo, go = R.pid_order(pids[:NQ]), R.pid_order(pids[NQ:])
args = (pids[:NQ], pids[NQ:], cams[:NQ], cams[NQ:])
L = N.lib()


def wall_and_device(fn, n=10):
    """(wall ms per call, device ms per call with the host running ahead of the GPU)."""
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / n * 1e3
    dev = []
    for _ in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(int(6e6))  # ~3 ms: the host enqueues the whole step behind it
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        dev.append(e0.elapsed_time(e1))
    return wall, sorted(dev)[len(dev) // 2]


cache = R.PlaneCache()
ids_u = R.encode_ids(*args, False, q.device)
ids_s = R.encode_ids(*args, False, q.device, q_order=qo, g_order=go)
for name, fn in {
    "step, caller order": lambda: R.topk_and_eval(R.build_planes(q), cache.get(g), 100, *args, ids=ids_u),
    "step, pid order, every tile": lambda: R.topk_and_eval(R.build_planes(q, order=qo), cache.get(g, order=go), 100, *args, ids=ids_s, tile_lists=False),
    "step, pid order, tile lists": lambda: R.topk_and_eval(R.build_planes(q, order=qo), cache.get(g, order=go), 100, *args, ids=ids_s),
    "topk only, subset threshold": lambda: R.topk(R.build_planes(q), cache.get(g), 100),
    "topk only, every tile": lambda: R.topk(R.build_planes(q), cache.get(g), 100, exact_threshold_pass=True),
    "evaluate_streamed, caller order": lambda: R.evaluate_streamed(R.build_planes(q), cache.get(g), *args, ids=ids_u),
    "evaluate_streamed, pid order": lambda: R.evaluate_streamed(R.build_planes(q, order=qo), cache.get(g, order=go), *args, ids=ids_s),
}.items():
    w, d = wall_and_device(fn)
    print(f"{name:40s} wall {w:.3f} ms   device {d:.3f} ms")

qp, gp = R.build_planes(q, order=qo), R.build_planes(g, order=go)
gmin = torch.empty(NQ, (NG + 15) // 16, device="cuda")
stride = L.ctl_dist_subset_stride(NG, 100)
work_pos = R._tile_list(qp, gp, ids_s, 0)
work_thr = R._tile_list(qp, gp, ids_s, stride)
torch.cuda.synchronize()
print(f"tiles: {(NQ + 127) // 128 * ((NG + 127) // 128)} total, {int(work_pos[0])} can hold a positive, {int(work_thr[0])} with stride {stride}")
ovf = torch.zeros(1, dtype=torch.int32, device="cuda")
pos_keys = torch.zeros(NQ, ids_s.max_pos, dtype=torch.int64, device="cuda")
pos_count = torch.zeros(NQ, dtype=torch.int32, device="cuda")
idk = dict(q_pid=ids_s.q_pid.data_ptr(), q_cam=ids_s.q_cam.data_ptr(), g_pid=ids_s.g_pid.data_ptr(),
           g_cammask=ids_s.g_mask.data_ptr(), max_pos=ids_s.max_pos, overflow=ovf.data_ptr(), g_index_map=gp.order.data_ptr())


def gpu_ms(desc, n=10):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    N.check(L.ctl_dist_pass(qp.ptr, NQ, gp.ptr, NG, D, qp.flags, C.byref(desc), N.stream_ptr()))
    e0.record()
    for _ in range(n):
        N.check(L.ctl_dist_pass(qp.ptr, NQ, gp.ptr, NG, D, qp.flags, C.byref(desc), N.stream_ptr()))
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def other_ms(fn, n=10):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


print("tile list kernel                       %.3f ms" % other_ms(lambda: R._tile_list(qp, gp, ids_s, stride)))
print("pass gmin, every tile                  %.3f ms" % gpu_ms(N.PassDesc(gmin=gmin.data_ptr())))
print("pass gmin + collect, every tile        %.3f ms" % gpu_ms(N.PassDesc(gmin=gmin.data_ptr(), pos_keys=pos_keys.data_ptr(), pos_count=pos_count.data_ptr(), **idk)))
print("pass gmin + collect, tile list         %.3f ms" % gpu_ms(N.PassDesc(gmin=gmin.data_ptr(), pos_keys=pos_keys.data_ptr(), pos_count=pos_count.data_ptr(), tile_list=work_thr.data_ptr(), **idk)))
print("pass collect only, tile list           %.3f ms" % gpu_ms(N.PassDesc(pos_keys=pos_keys.data_ptr(), pos_count=pos_count.data_ptr(), tile_list=work_pos.data_ptr(), **idk)))
# pass 2 of the step with the two thresholds (candidate volume)
pos_count.zero_()
N.check(L.ctl_dist_pass(qp.ptr, NQ, gp.ptr, NG, D, qp.flags, C.byref(N.PassDesc(pos_keys=pos_keys.data_ptr(), pos_count=pos_count.data_ptr(), **idk)), N.stream_ptr()))
N.check(L.ctl_sort_key_rows(pos_keys.data_ptr(), pos_count.data_ptr(), NQ, ids_s.max_pos, N.stream_ptr()))
buckets = torch.zeros(NQ, ids_s.max_pos + 1, dtype=torch.int32, device="cuda")
cand = torch.empty(NQ, 4096, dtype=torch.int64, device="cuda")
cc = torch.zeros(NQ, dtype=torch.int32, device="cuda")
tau = torch.empty(NQ, device="cuda")
for name, wl in (("every tile", None), ("tile list", work_thr)):
    gmin.fill_(float("inf"))
    N.check(L.ctl_dist_pass(qp.ptr, NQ, gp.ptr, NG, D, qp.flags, C.byref(N.PassDesc(gmin=gmin.data_ptr(), tile_list=N.ptr(wl))), N.stream_ptr()))
    N.check(L.ctl_select_tau(gmin.data_ptr(), NQ, (NG + 15) // 16, 1, 100, tau.data_ptr(), N.stream_ptr()))
    cc.zero_()
    d2 = N.PassDesc(tau=tau.data_ptr(), cand_keys=cand.data_ptr(), cand_count=cc.data_ptr(), cand_cap=4096, thr_keys=pos_keys.data_ptr(),
                    thr_count=pos_count.data_ptr(), buckets=buckets.data_ptr(), **idk)
    N.check(L.ctl_dist_pass(qp.ptr, NQ, gp.ptr, NG, D, qp.flags, C.byref(d2), N.stream_ptr()))
    torch.cuda.synchronize()
    c = cc.float()
    print(f"threshold from {name:10s}: candidates per query mean {c.mean().item():.0f}, max {c.max().item():.0f}; "
          f"pass 2 {gpu_ms(d2):.3f} ms (counts keep growing: timing only); sort {other_ms(lambda: L.ctl_sort_key_rows(cand.data_ptr(), cc.data_ptr(), NQ, 4096, N.stream_ptr())):.3f} ms")
    cc.clamp_(max=4096)
