"""Needs a GPU: wall-time breakdown of one retrieval step (3368 x 15913 x 2048, top-100 + CMC/mAP)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import ctl_b200
from ctl_b200 import retrieval as R, synth

feats, pids, cams = synth.synth_retrieval(3368, 15913, 751, 2048, 3.0, 0)
q, g = feats[:3368].cuda(), feats[3368:].cuda()
def T(fn, n=5):
    fn(); torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n): fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e3
print("build_planes q+g        %.3f ms" % T(lambda: (R.build_planes(q), R.build_planes(g))))
qp, gp = R.build_planes(q), R.build_planes(g)
print("encode_identities (host) %.3f ms" % T(lambda: R.encode_identities(pids[:3368], pids[3368:], cams[:3368], cams[3368:], False)))
print("topk only (2 passes)     %.3f ms" % T(lambda: R.topk(qp, gp, 100)))
print("evaluate_streamed        %.3f ms" % T(lambda: R.evaluate_streamed(qp, gp, pids[:3368], pids[3368:], cams[:3368], cams[3368:])))
print("topk_and_eval (fused)    %.3f ms" % T(lambda: R.topk_and_eval(qp, gp, 100, pids[:3368], pids[3368:], cams[:3368], cams[3368:])))
print("max_pos probe"); ids = R.encode_ids(pids[:3368], pids[3368:], cams[:3368], cams[3368:], False, q.device)
print("max_pos =", ids.max_pos); print("evaluate_streamed (ids cached) %.3f ms" % T(lambda: R.evaluate_streamed(qp, gp, pids[:3368], pids[3368:], cams[:3368], cams[3368:], ids=ids)))
print("topk_and_eval (ids cached)     %.3f ms" % T(lambda: R.topk_and_eval(qp, gp, 100, pids[:3368], pids[3368:], cams[:3368], cams[3368:], ids=ids)))
import ctypes as C
from ctl_b200 import _native as N
L = N.lib()
nq, ng = 3368, 15913
gmin = torch.empty(nq, (ng + 15) // 16, device="cuda")
def gpu_ms(desc, n=10):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    N.check(L.ctl_dist_pass(qp.ptr, nq, gp.ptr, ng, 2048, qp.flags, C.byref(desc), N.stream_ptr()))
    e0.record()
    for _ in range(n):
        N.check(L.ctl_dist_pass(qp.ptr, nq, gp.ptr, ng, 2048, qp.flags, C.byref(desc), N.stream_ptr()))
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n
idk = dict(q_pid=ids.q_pid.data_ptr(), q_cam=ids.q_cam.data_ptr(), g_pid=ids.g_pid.data_ptr(), g_cammask=ids.g_mask.data_ptr(), max_pos=ids.max_pos)
ovf = torch.zeros(1, dtype=torch.int32, device="cuda")
pos_keys = torch.zeros(nq, ids.max_pos, dtype=torch.int64, device="cuda"); pos_count = torch.zeros(nq, dtype=torch.int32, device="cuda")
print("pass gmin only            %.3f ms" % gpu_ms(N.PassDesc(gmin=gmin.data_ptr())))
print("pass gmin + collect       %.3f ms (counts overflow after the 1st call; timing only)" % gpu_ms(N.PassDesc(gmin=gmin.data_ptr(), pos_keys=pos_keys.data_ptr(), pos_count=pos_count.data_ptr(), overflow=ovf.data_ptr(), **idk)))
pos_count.zero_()
N.check(L.ctl_dist_pass(qp.ptr, nq, gp.ptr, ng, 2048, qp.flags, C.byref(N.PassDesc(pos_keys=pos_keys.data_ptr(), pos_count=pos_count.data_ptr(), overflow=ovf.data_ptr(), **idk)), N.stream_ptr()))
N.check(L.ctl_sort_key_rows(pos_keys.data_ptr(), pos_count.data_ptr(), nq, ids.max_pos, N.stream_ptr()))
buckets = torch.zeros(nq, ids.max_pos + 1, dtype=torch.int32, device="cuda")
print("pass count                %.3f ms" % gpu_ms(N.PassDesc(thr_keys=pos_keys.data_ptr(), thr_count=pos_count.data_ptr(), buckets=buckets.data_ptr(), **idk)))
tau = torch.full((nq,), 1.9, device="cuda"); cand = torch.empty(nq, 4096, dtype=torch.int64, device="cuda"); cc = torch.zeros(nq, dtype=torch.int32, device="cuda")
print("pass cand(tau=1.9)+count  %.3f ms" % gpu_ms(N.PassDesc(tau=tau.data_ptr(), cand_keys=cand.data_ptr(), cand_count=cc.data_ptr(), cand_cap=4096, overflow=ovf.data_ptr(), thr_keys=pos_keys.data_ptr(), thr_count=pos_count.data_ptr(), buckets=buckets.data_ptr(), **idk)))
print("dist_matrix (1 pass)     %.3f ms" % T(lambda: R.dist_matrix(q, g)))
