"""Needs a GPU: epilogue phase counters of pass 2 (candidates + bucket counts) in caller order vs identity order."""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import ctl_b200  # noqa: F401
from ctl_b200 import _native as N
from ctl_b200 import retrieval as R
from ctl_b200 import synth

NQ, NG, D, K = 3368, 15913, 2048, 100
feats, pids, cams = synth.synth_retrieval(NQ, NG, 751, D, 3.0, 0)
q, g = feats[:NQ].cuda(), feats[NQ:].cuda()
args = (pids[:NQ], pids[NQ:], cams[:NQ], cams[NQ:])
L = N.lib()
PH = ["tile_setup", "mma_and_stage", "bar_meta", "acc_read", "element_loop", "tile_end"]


def run(name, qp, gp, ids, gmap):
    n_groups = (NG + 15) // 16
    gmin = torch.empty(NQ, n_groups, device="cuda")
    tau = torch.empty(NQ, device="cuda")
    ovf = torch.zeros(1, dtype=torch.int32, device="cuda")
    pos = torch.zeros(NQ, ids.max_pos, dtype=torch.int64, device="cuda")
    cnt = torch.zeros(NQ, dtype=torch.int32, device="cuda")
    idk = dict(q_pid=ids.q_pid.data_ptr(), q_cam=ids.q_cam.data_ptr(), g_pid=ids.g_pid.data_ptr(), g_cammask=ids.g_mask.data_ptr(),
               max_pos=ids.max_pos, overflow=ovf.data_ptr(), g_index_map=N.ptr(gmap))
    s = N.stream_ptr
    N.check(L.ctl_dist_pass(qp.ptr, NQ, gp.ptr, NG, D, qp.flags, C.byref(N.PassDesc(gmin=gmin.data_ptr(), pos_keys=pos.data_ptr(), pos_count=cnt.data_ptr(), **idk)), s()))
    N.check(L.ctl_select_tau(gmin.data_ptr(), NQ, n_groups, 1, K, tau.data_ptr(), s()))
    N.check(L.ctl_sort_key_rows(pos.data_ptr(), cnt.data_ptr(), NQ, ids.max_pos, s()))
    for what in ("cand+count", "count only", "cand only"):
        times = []
        for rep in range(4):
            cand = torch.empty(NQ, 4096, dtype=torch.int64, device="cuda")
            cc = torch.zeros(NQ, dtype=torch.int32, device="cuda")
            buckets = torch.zeros(NQ, ids.max_pos + 1, dtype=torch.int32, device="cuda")
            d = N.PassDesc(**idk)
            if what != "count only":
                d.tau, d.cand_keys, d.cand_count, d.cand_cap = tau.data_ptr(), cand.data_ptr(), cc.data_ptr(), 4096
            if what != "cand only":
                d.thr_keys, d.thr_count, d.buckets = pos.data_ptr(), cnt.data_ptr(), buckets.data_ptr()
            prof = torch.zeros(148 * 2 * 8, dtype=torch.int64, device="cuda")
            if rep == 3:
                L.ctl_debug_set_dist_profile(prof.data_ptr())
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            N.check(L.ctl_dist_pass(qp.ptr, NQ, gp.ptr, NG, D, qp.flags, C.byref(d), s()))
            e1.record()
            torch.cuda.synchronize()
            L.ctl_debug_set_dist_profile(None)
            times.append(e0.elapsed_time(e1))
        pm = prof.view(148, 2, 8).double()
        tot = pm[:, 0, :6].sum(1)
        print(f"{name:12s} {what:11s} {min(times[:3]):.3f} ms | mean/CTA:", ", ".join(f"{PH[i]}={pm[:, 0, i].mean().item():.0f}" for i in range(6)),
              f"| element_loop per CTA min {pm[:, 0, 4].min().item():.0f} max {pm[:, 0, 4].max().item():.0f}; total per CTA min {tot.min().item():.0f} max {tot.max().item():.0f}",
              f"| cand/query mean {cc.float().mean().item():.0f}" if what != "count only" else "")


ids_u = R.encode_ids(*args, False, q.device)
run("caller order", R.build_planes(q), R.build_planes(g), ids_u, None)
qo, go = R.pid_order(pids[:NQ]), R.pid_order(pids[NQ:])
ids_s = R.encode_ids(*args, False, q.device, q_order=qo, g_order=go)
gp = R.build_planes(g, order=go)
run("pid order", R.build_planes(q, order=qo), gp, ids_s, gp.order)
ids_g = R.encode_ids(*args, False, q.device, g_order=go)
run("gallery only", R.build_planes(q), gp, ids_g, gp.order)
