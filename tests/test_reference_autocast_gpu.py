"""Same-precision parity AT THE BENCH SHAPES against the UNMODIFIED reference executed on a GPU.

The reference's own trunk modules (modelling/backbones/resnet.py:122-133, resnet_ibn_a.py:126-141,
modelling/baseline.py:91-96) were run on cuda:0 under ``torch.autocast(dtype=float16)`` -- the precision the reference's
configs train and validate at (USE_MIXED_PRECISION -> PL native AMP, utils/misc.py:111) -- and in fp32 by
``python -m oracle.make_golden --only bench_autocast``; tests/golden/bench_autocast_*.npz hold what these tests compare
against (inputs are regenerated from the same seeds and checked by checksum):

  * the eval embedding at metric M1's configuration (256 crops of 256x128, ResNet50) and at config 4's per-GPU eval shape
    (128 crops of 320x320, ResNet50-IBN-a): every 16th image, tolerance 2e-3 of the feature scale (two correct fp16
    evaluations of this network differ by a few 1e-4; the reference's own autocast run is 4-7e-4 away from its fp32
    run, tests/golden/trunk_autocast.npz);
  * one training step at config 2's shape (16 ids x 16 instances of 256x128) and config 4's per-GPU shape (32 x 4 of
    320x320, IBN-a): train-mode features of every 16th image within 2e-2, every parameter gradient by direction (cosine
    >= 0.95 against BOTH the reference's autocast and fp32 gradients on a fixed, evenly strided sample of 512 elements
    per tensor) and size (full norm within 6 %): ReLU masks make element-wise comparison of two fp16 backward passes
    meaningless.
"""
import numpy as np
import pytest
import torch

from oracle import ctl_oracle as O
from conftest import load_golden

pytestmark = pytest.mark.gpu

ROW_STRIDE, GRAD_SAMPLE = 16, 512  # oracle/make_golden.py: BENCH_ROW_STRIDE, BENCH_GRAD_SAMPLE


def _checksum(t):
    t = torch.as_tensor(t).double()
    return np.array([float(t.sum()), float((t * t).sum())])


def _sample(t):
    f = t.detach().flatten()
    return f[:: max(1, f.numel() // GRAD_SAMPLE)][:GRAD_SAMPLE]


@pytest.mark.parametrize("tag,ibn,hw,bs", [("r50", False, (256, 128), 256), ("ibn", True, (320, 320), 128)])
def test_eval_embedding_at_bench_shape_vs_reference_cuda_autocast(tag, ibn, hw, bs):
    from ctl_b200.modelling.backbones.engine import TrunkEngine

    g = load_golden(f"bench_autocast_eval_{tag}.npz")
    sd = O.make_trunk_state(seed=7, ibn=ibn)
    x = torch.randn(bs, 3, *hw, generator=torch.Generator().manual_seed(77))
    np.testing.assert_allclose(_checksum(x), g["in_checksum"], rtol=1e-9)
    f32, amp = torch.from_numpy(g["feat_fp32"]), torch.from_numpy(g["feat_amp"])
    feat = TrunkEngine(sd, "cuda", ibn=ibn).forward(x.cuda())["global_feat"][::ROW_STRIDE].cpu()
    scale = float(f32.abs().max())
    e_amp = float((feat - amp).abs().max()) / scale
    e_f32 = float((feat - f32).abs().max()) / scale
    own = float((amp - f32).abs().max()) / scale
    print(f"{tag} bs {bs} {hw}: engine vs reference CUDA-autocast {e_amp:.3e}; engine vs reference fp32 {e_f32:.3e}; "
          f"reference CUDA-autocast vs its own fp32 {own:.3e}")
    assert torch.isfinite(feat).all()
    assert e_amp <= 2e-3
    assert e_f32 <= max(3.0 * own, 1.5e-3)


# Margin note (measured on an H100 80GB HBM3): at config 4 the norm check of the IBN-a InstanceNorm bias gradients sits
# close to its 6 % bound.  Those gradients are sums over ~800k positions that almost cancel, so last-bit changes to any
# training kernel move them through the ReLU masks: the reference's own autocast run is up to 4.5 % from its fp32 run on
# them, and of two equally valid BatchNorm pivot rows the first put layer1.0.bn1.IN.bias at 6.7 % while the last (the
# committed kernel) passes.  A failure here after a change of rounding is not by itself a wrong kernel;
# check the change against float64 first (tests/test_train_kernels_gpu.py), and do not pick numerics by this outcome.
@pytest.mark.parametrize("tag,ibn,hw,P,K", [("r50 cfg2", False, (256, 128), 16, 16), ("ibn cfg4/gpu", True, (320, 320), 32, 4)])
def test_training_step_at_bench_shape_vs_reference_cuda_autocast(tag, ibn, hw, P, K):
    from ctl_b200.modelling.backbones.engine_train import TrunkTrainer

    g = load_golden(f"bench_autocast_train_{'ibn' if ibn else 'r50'}.npz")
    n = P * K
    scale = 1024.0
    sd = O.make_trunk_state(seed=17, ibn=ibn)
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(n, 3, *hw, generator=gen)
    dfeat = torch.randn(n, 2048, generator=gen) * 1e-3
    np.testing.assert_allclose(_checksum(torch.cat((x.flatten(), dfeat.flatten()))), g["in_checksum"], rtol=1e-9)
    params = {k: v.clone().cuda() for k, v in sd.items() if v.is_floating_point()}
    tr = TrunkTrainer("cuda", grad_scale=scale, ibn=ibn)
    feat = tr.forward(x.cuda(), params)
    grads = tr.backward(dfeat.cuda())
    torch.cuda.synchronize()
    rfeat = torch.from_numpy(g["feat_amp"])
    fscale = float(rfeat.abs().max())
    e = float((feat[::ROW_STRIDE].cpu() - rfeat).abs().max()) / fscale

    def cos(a_, b_):
        return float((a_ * b_).sum() / (a_.norm() * b_.norm() + 1e-300))

    names = [str(k) for k in g["names"]]
    worst_cos, worst_norm, unresolved = (1.0, None), (0.0, None), []
    for k in names:
        gk = grads[k].double()
        assert torch.isfinite(gk).all(), k
        rg_norm, r32_norm, ref_cos = (float(v) for v in g[f"stats/{k}"])
        if ref_cos < 0.9:  # the reference under autocast does not reproduce its own fp32 gradient here
            unresolved.append(k)
            partner = grads.get(k[:-4] + "weight") if k.endswith("bias") else None
            bound = 3.0 * max(rg_norm, r32_norm) + (2e-2 * float(partner.double().norm()) if partner is not None else 0.0)
            assert float(gk.norm()) <= bound + 1e-12, (k, float(gk.norm()), bound)  # round-off sized, like the reference's
            continue
        gs = _sample(gk).cpu()
        rg, r32 = torch.from_numpy(g[f"amp/{k}"]).double(), torch.from_numpy(g[f"fp32/{k}"]).double()
        c = min(cos(gs, rg), cos(gs, r32))
        nr = abs(float(gk.norm()) / rg_norm - 1)
        if c < worst_cos[0]:
            worst_cos = (c, k)
        if nr > worst_norm[0]:
            worst_norm = (nr, k)
    print(f"{tag}: gradients the reference's own autocast run does not resolve (cos < 0.9 vs its fp32 run): {unresolved}")
    assert len(unresolved) <= 4, unresolved
    print(f"{tag}: train features vs reference CUDA-autocast {e:.3e}; worst gradient cosine {worst_cos[0]:.4f} "
          f"({worst_cos[1]}), worst norm deviation {worst_norm[0]:.3e} ({worst_norm[1]}) over {len(names)} tensors")
    assert e <= 2e-2
    assert worst_cos[0] >= 0.95, worst_cos
    assert worst_norm[0] <= 6e-2, worst_norm
