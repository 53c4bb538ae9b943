"""Needs a GPU; test-side debugging aid (executes the oracle like tests/ do): per-parameter gradient error of the training
trunk vs the float64 oracle, for several loss scales."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import ctl_b200
from oracle import ctl_oracle as O
from ctl_b200.modelling.backbones.engine_train import TrunkTrainer

sd = O.make_trunk_state(seed=7)
g = torch.Generator().manual_seed(1)
n, H, W = 8, 128, 64
x = torch.randn(n, 3, H, W, generator=g)
dfeat = torch.randn(n, 2048, generator=g) * 1e-3
feat_o, grads_o, _ = O.trunk_train_fp16sim(x, sd, dfeat)
gmax = max(float(v.abs().max()) for v in grads_o.values())
for scale in [float(s) for s in sys.argv[1:]] or [4096.0]:
    params = {k: v.clone().cuda() for k, v in sd.items() if v.is_floating_point()}
    tr = TrunkTrainer("cuda", grad_scale=scale)
    feat = tr.forward(x.cuda(), params)
    grads = tr.backward(dfeat.cuda())
    torch.cuda.synchronize()
    print(f"== grad_scale {scale}: feat rel err {float((feat.cpu().double()-feat_o).abs().max()/feat_o.abs().max()):.3e}")
    for k in grads_o:
        go, gk = grads_o[k], grads[k].cpu().double()
        rel = float((gk - go).abs().max() / (go.abs().max() + 1e-30))
        cos = float((gk * go).sum() / (gk.norm() * go.norm() + 1e-30))
        if "conv" in k or "downsample.0" in k or k.endswith("bn3.weight"):
            print(f"  {k:34s} rel {rel:9.3e} cos {cos:8.5f} |ref| {float(go.abs().max()):9.3e} ratio {float(gk.norm()/(go.norm()+1e-30)):.4f}")
