"""The base model's training step (train_base_model.py:38-96) on the GPU.

Line 1, the loss step alone at B = 256 (16 ids x 16, a quarter of the ids padded with mock rows), D = 2048, C = 751:
  - fused eager: BaseStepFn forward + backward (one ctl_base_loss_step enqueue plus the autograd bookkeeping);
  - fused graph: replay of a captured ctl_base_loss_step;
  - composed: the same arithmetic from the stand-alone drop-ins (TripletLoss, CenterLoss, torch BatchNorm1d + bias-free
    Linear, CrossEntropyLabelSmooth), forward + backward.  CenterLoss reads its loss back to check the label range, so
    this path synchronises once per call.
Line 2, one full iteration at 16 x 16 crops of 256x128 (ResNet50 train-mode trunk forward and backward, loss, fused Adam
  + center SGD, the one read-back of the logged parts): BaseModel.training_step and CTLModel.training_step with their
  optimizers attached, alternating window by window in the same process so that both see the same clocks.
Every time is the median of --reps windows, with the windows' min and max beside it.  Both lines carry the card's name
and power limit.

    python tools/bench_base_train.py [--iters 50] [--train-iters 5] [--reps 5] [--loss-only]
"""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import ctl_b200  # noqa: E402,F401
from ctl_b200 import _native as N  # noqa: E402
from ctl_b200.losses._fn import BaseStepFn  # noqa: E402
from ctl_b200.losses.center_loss import CenterLoss  # noqa: E402
from ctl_b200.losses.triplet_loss import CrossEntropyLabelSmooth, TripletLoss  # noqa: E402
from oracle import ctl_oracle as O  # noqa: E402
from tools.bench_basic import card, graphed, spread, time_ms  # noqa: E402

NUM_CLASSES, DIM = 751, 2048


def _line(prefix, t):
    return {f"{prefix}_ms": round(t[0], 4), f"{prefix}_min_max": spread(t)}


def loss_step(iters, reps):
    P, K = 16, 16
    B = P * K
    feats, labels, is_real = O.synth_batch(P, K, DIM, NUM_CLASSES, seed=4, pad_fraction=0.25, scale=0.5)
    g = torch.Generator().manual_seed(1004)
    f = feats.cuda()
    lab, real = labels.cuda(), is_real.cuda()
    centers = torch.randn(NUM_CLASSES, DIM, generator=g).cuda()
    bn_w = (0.5 + torch.rand(DIM, generator=g)).cuda()
    bn_b = torch.zeros(DIM, device="cuda")
    fc_w = (0.02 * torch.randn(NUM_CLASSES, DIM, generator=g)).cuda()
    rm, rv = torch.zeros(DIM, device="cuda"), torch.ones(DIM, device="cuda")
    cfg = N.BaseLossConfig(B, DIM, NUM_CLASSES, 0.5, 0, 0, 5e-4, 1.0, 1.0, 1e-5, 0.1, 0.1)
    leaves = [t.clone().requires_grad_(True) for t in (f, centers, bn_w, fc_w)]

    def fused_eager():
        for t in leaves:
            t.grad = None
        total, _ = BaseStepFn.apply(*leaves, bn_b, rm, rv, lab, real, cfg)
        total.backward()

    L = N.lib()
    lab32, real8 = lab.int(), real.to(torch.uint8)
    out = torch.zeros(6, device="cuda")
    grads = [torch.empty_like(t) for t in (f, centers, bn_w, fc_w)]
    ws = torch.empty(L.ctl_base_loss_workspace_bytes(C.byref(cfg)), dtype=torch.uint8, device="cuda")

    def fused_raw():
        N.check(L.ctl_base_loss_step(C.byref(cfg), f.data_ptr(), lab32.data_ptr(), real8.data_ptr(), centers.data_ptr(),
                                     bn_w.data_ptr(), bn_b.data_ptr(), rm.data_ptr(), rv.data_ptr(), fc_w.data_ptr(),
                                     out.data_ptr(), grads[0].data_ptr(), grads[1].data_ptr(), grads[2].data_ptr(),
                                     grads[3].data_ptr(), ws.data_ptr(), ws.numel(), N.stream_ptr()))

    trip = TripletLoss(0.5, "euclidean")
    cl = CenterLoss(NUM_CLASSES, DIM).cuda()
    bn = torch.nn.BatchNorm1d(DIM).cuda().train()
    bn.bias.requires_grad_(False)
    fc = torch.nn.Linear(DIM, NUM_CLASSES, bias=False).cuda()
    xent = CrossEntropyLabelSmooth(NUM_CLASSES)
    with torch.no_grad():
        cl.centers.copy_(centers)
        bn.weight.copy_(bn_w)
        fc.weight.copy_(fc_w)
    fc_in = f.clone().requires_grad_(True)
    mods = (cl, bn, fc)

    def composed():
        fc_in.grad = None
        for m in mods:
            m.zero_grad(set_to_none=True)
        lq, _, _ = trip(fc_in, lab, mask=real)
        total = 5e-4 * cl(fc_in, lab) + xent(fc(bn(fc_in)), lab) + lq
        total.backward()

    eager = time_ms(fused_eager, iters, reps)
    graph = time_ms(graphed(fused_raw), iters, reps)
    comp = time_ms(composed, iters, reps)
    line = {"what": "base loss step, B=256 D=2048 C=751, forward + backward", "iters": iters, "reps": reps}
    line.update(_line("fused_eager", eager))
    line.update(_line("fused_graph", graph))
    line.update(_line("composed_drop_ins", comp))
    line["composed_over_fused_eager"] = round(comp[0] / eager[0], 2)
    return line


class _Cfg(dict):
    __getattr__ = dict.__getitem__


def _train_cfg():
    """bench.py's training configuration (config 2: ResNet50, Adam, center SGD, dynamic loss scaling), past warm-up."""
    return _Cfg(MODEL=_Cfg(NAME="resnet50", LAST_STRIDE=1, PRETRAINED=False, PRETRAIN_PATH="", BACKBONE_EMB_SIZE=DIM,
                           USE_CENTROIDS=False, KEEP_CAMID_CENTROIDS=True, RESUME_TRAINING=False),
                SOLVER=_Cfg(MARGIN=0.5, DISTANCE_FUNC="euclidean", CENTER_LOSS_WEIGHT=5e-4, QUERY_XENT_WEIGHT=1.0,
                            QUERY_CONTRASTIVE_WEIGHT=1.0, CENTROID_CONTRASTIVE_WEIGHT=1.0, OPTIMIZER_NAME="Adam",
                            BASE_LR=1e-4, WEIGHT_DECAY=5e-4, CENTER_LR=0.5, LR_SCHEDULER_NAME="multistep_lr",
                            LR_STEPS=(40, 70), GAMMA=0.1, USE_WARMUP_LR=False, WARMUP_EPOCHS=10),
                DATALOADER=_Cfg(NUM_INSTANCE=16), TEST=_Cfg(FEAT_NORM=True, ONLY_TEST=False, VISUALIZE="no"),
                USE_MIXED_PRECISION=True)


def full_iteration(iters, reps):
    from ctl_b200.modelling.base_model import BaseModel
    from ctl_b200.modelling.ctl_model import CTLModel

    P, K = 16, 16
    g = torch.Generator().manual_seed(1234)
    x = torch.randn(P * K, 3, 256, 128, generator=g).cuda()
    labels = torch.arange(P).repeat_interleave(K).cuda()
    batch = (x, labels, torch.zeros(P * K, dtype=torch.long).cuda(), torch.ones(P * K, dtype=torch.bool).cuda())
    models = {}
    for name, cls in (("base", BaseModel), ("ctl", CTLModel)):
        torch.manual_seed(0)
        m = cls(_train_cfg(), num_classes=NUM_CLASSES, num_query=0).cuda().train()
        (opt, opt_center), _ = m.configure_optimizers()
        m.attach_optimizers(opt, opt_center)
        for _ in range(3):
            m.training_step(batch, 0)
        models[name] = m
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = {k: [] for k in models}
    losses = {}
    for _ in range(reps):
        for name, m in models.items():  # alternate: base window, CTL window, base window, ...
            e0.record()
            for _ in range(iters):
                out = m.training_step(batch, 0)
            e1.record()
            torch.cuda.synchronize()
            ts[name].append(e0.elapsed_time(e1) / iters)
            losses[name] = float(out["loss"])
    line = {"what": "full iteration, ResNet50 16x16 crops of 256x128: trunk fwd+bwd, loss, Adam, center SGD",
            "iters": iters, "reps": reps}
    for name, t in ts.items():
        t.sort()
        med = t[len(t) // 2]
        line.update(_line(f"{name}_iteration", (med, t[0], t[-1])))
        line[f"{name}_images_per_s"] = round(P * K / med * 1e3, 1)
        line[f"{name}_last_loss"] = round(losses[name], 4)
    line["peak_mem_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50, help="loss-step calls per window")
    ap.add_argument("--train-iters", type=int, default=5, help="full iterations per window")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--loss-only", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_base_train.py needs a GPU"
    name, power = card()
    head = {"gpu": name, "power_limit": power}
    print(json.dumps({**head, **loss_step(args.iters, args.reps)}), flush=True)
    if not args.loss_only:
        print(json.dumps({**head, **full_iteration(args.train_iters, args.reps)}), flush=True)


if __name__ == "__main__":
    main()
