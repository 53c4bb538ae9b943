"""TEST INFRASTRUCTURE ONLY -- CPU oracle of the base model's training-step losses (train_base_model.py:38-96, the
paper's baseline without centroid rounds) and the generator of tests/golden/base_loss_*.npz.

    python -m oracle.base_oracle      runs the UNMODIFIED reference's train_base_model.CTLModel.training_step on the CPU
                                      (oracle/ref_import.py stubs, make_golden's _FixedTrunk / _Trainer stand-ins) and
                                      writes tests/golden/base_loss_{case}.npz for every LOSS_CASES and LOSS_VARIANTS case;
                                      those files pin this module (tests/test_base_model_cpu.py)

Like oracle/basic_oracle.py, this module stands beside oracle/ctl_oracle.py and oracle/make_golden.py instead of adding
to them: those files pin the CTL step and every existing golden, and they are kept byte-for-byte as they were.  The
inputs and head state are make_golden's gen_loss ones, so a base_loss_* file and the loss_* file of the same case share
their inputs.  The scalars (minus `ctl` and `l2_centroid`, which the base step does not have) and the BatchNorm vectors
are stored whole; the [B, D] feature gradient and the [C, D] center / fc gradients are stored as a row sample
(`golden_rows`: every mock row up to half the sample, the rest evenly strided; the center / fc rows of those rows'
labels) next to checksums of the whole tensors, which keeps every file a few hundred kB.

Only tests/ and tools/ may import this module; the product never does.
"""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ctl_oracle as O  # noqa: E402
from oracle.make_golden import (DIM, GOLD, LOSS_CASES, LOSS_VARIANTS, NUM_CLASSES, _FixedTrunk, _Trainer,  # noqa: E402
                                checksum, head_state)

# every golden case: name -> ((P, K, pad_fraction, seed, scale), SOLVER overrides)
BASE_CASES = {**{k: (v, {}) for k, v in LOSS_CASES.items()},
              **{k: (LOSS_CASES[b], o) for k, (b, o) in LOSS_VARIANTS.items()}}


def base_step_losses(
    feats: torch.Tensor,
    labels: torch.Tensor,
    is_real: torch.Tensor,
    centers: torch.Tensor,
    bn_weight: torch.Tensor,
    bn_bias: torch.Tensor,
    fc_weight: torch.Tensor,
    *,
    margin=0.5,
    center_loss_weight=5e-4,
    query_xent_weight=1.0,
    query_contrastive_weight=1.0,
    bn_eps=1e-5,
    bn_momentum=0.1,
    epsilon=0.1,
    dist_func="euclidean",
    running_mean=None,
    running_var=None,
):
    """Everything the base model's training_step computes after the trunk and before backward
    (train_base_model.py:57-75) as a differentiable torch-CPU function of (feats, centers, bn_weight, fc_weight); float64
    inputs give a float64 checker.  running_mean / running_var (optional) are updated in place like nn.BatchNorm1d's.

    Returns dict(total, xent, triplet, center, dist_ap, dist_an)."""
    is_real = is_real.bool()
    # :60-65 query triplet: distances and batch-hard mining over ALL rows, then anchors masked to isReal
    l_q, ap, an = O.triplet_loss(feats, labels, margin, mask=is_real, dist_func=dist_func)
    l_q = l_q * query_contrastive_weight
    # :67-69 center loss over ALL rows, mock rows included
    l_cen = center_loss_weight * O.center_loss(feats, labels, centers)
    # :70-73 BatchNorm1d (batch statistics over ALL rows) -> bias-free fc_query -> label-smoothed CE over ALL rows
    bn_f = F.batch_norm(feats, running_mean, running_var, bn_weight, bn_bias, True, bn_momentum, bn_eps)
    logits = bn_f @ fc_weight.t()
    l_x = O.cross_entropy_label_smooth(logits, labels, fc_weight.shape[0], epsilon) * query_xent_weight
    total = l_cen + l_x + l_q  # :75
    # :91-94 logged means of the masked (real-anchor) distances
    return dict(total=total, xent=l_x, triplet=l_q, center=l_cen, dist_ap=ap.detach().mean(),
                dist_an=an.detach().mean())


GOLDEN_FEAT_ROWS = 16   # stored rows of the feature gradient
GOLDEN_LABEL_ROWS = 8   # stored rows of the center / fc gradients


def golden_rows(labels, is_real):
    """(feature rows, labels) whose gradient rows a golden stores: the mock rows first (their center-loss and head
    gradients are what sets the base step apart from the CTL step), up to half of GOLDEN_FEAT_ROWS, then evenly strided
    rows; the labels of those rows, mock rows' first, up to GOLDEN_LABEL_ROWS.  Both sorted ascending."""
    labels, is_real = np.asarray(labels), np.asarray(is_real, dtype=bool)
    B = len(labels)
    mock = np.flatnonzero(~is_real)[: GOLDEN_FEAT_ROWS // 2]
    strided = np.linspace(0, B - 1, GOLDEN_FEAT_ROWS - len(mock)).round().astype(np.int64)
    rows = np.unique(np.concatenate([mock, strided]))
    labs = list(dict.fromkeys(labels[mock].tolist() + labels[strided].tolist()))[:GOLDEN_LABEL_ROWS]
    return rows, np.sort(np.asarray(labs, dtype=np.int64))


def load_train_base(ref):
    """The reference's train_base_model module, imported in place next to the modules oracle/ref_import.py loaded (its
    `config`, `modelling.bases` and `utils` imports resolve to those)."""
    from oracle.ref_import import REFERENCE_ROOT

    if "train_base_model" in sys.modules:
        return sys.modules["train_base_model"]
    sys.path.insert(0, REFERENCE_ROOT)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            import train_base_model
    finally:
        sys.path.remove(REFERENCE_ROOT)
    return train_base_model


def generate():
    from oracle.ref_import import default_cfg, load_reference

    torch.set_num_threads(os.cpu_count())
    ref = load_reference()
    train_base = load_train_base(ref)
    for name, ((P, K, pad, seed, scale), solver_over) in BASE_CASES.items():
        feats, labels, is_real = O.synth_batch(P, K, DIM, NUM_CLASSES, seed, pad, scale)
        hs = head_state(seed)
        cfg = default_cfg(ref)
        cfg.DATALOADER.NUM_INSTANCE = K
        for k_, v_ in solver_over.items():
            cfg.SOLVER[k_] = v_
        model = train_base.CTLModel(cfg, num_classes=NUM_CLASSES, num_query=1)
        model.backbone = _FixedTrunk(feats)
        with torch.no_grad():
            model.center_loss.centers.copy_(hs["centers"])
            model.bn.weight.copy_(hs["bn_weight"])
            model.bn.bias.copy_(hs["bn_bias"])
            model.fc_query.weight.copy_(hs["fc_weight"])
        model.trainer = _Trainer()
        params = [p for n, p in model.named_parameters() if "center" not in n and p.requires_grad]
        opt = torch.optim.SGD(params, lr=0.0)
        opt_c = torch.optim.SGD(model.center_loss.parameters(), lr=0.0)
        model._ctl_optimizers = (opt, opt_c)
        model.train()
        x = torch.zeros(P * K, 3, 8, 8)
        cam = torch.zeros(P * K, dtype=torch.long)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out = model.training_step((x, labels, cam, is_real), 0)
        parts = {n: model.losses_dict[n][-1] for n in model.losses_names if model.losses_dict[n]}
        assert model.losses_dict["centroid_triplet"] == []  # train_base_model.py:88-89 zips 4 names with 3 values
        gf = model.backbone.feats.grad
        rows, labs = golden_rows(labels.numpy(), is_real.numpy())
        labs = torch.from_numpy(labs)
        np.savez_compressed(
            os.path.join(GOLD, f"base_loss_{name}.npz"),
            P=P, K=K, pad=pad, seed=seed, scale=scale,
            in_checksum=checksum(feats),
            is_real=is_real.numpy(),
            labels=labels.numpy(),
            total=float(out["loss"]),
            xent=parts["query_xent"], triplet=parts["query_triplet"], center=parts["query_center"],
            dist_ap=out["other"]["step_dist_ap"], dist_an=out["other"]["step_dist_an"],
            grad_feats_rows=gf[rows].numpy(),
            grad_feats_rows_idx=rows,
            grad_feats_checksum=checksum(gf),
            grad_feats_abs_max=float(gf.abs().max()),
            # NB: after training_step the reference has multiplied centers.grad by
            # 1/CENTER_LOSS_WEIGHT (train_base_model.py:80-81); stored as seen by opt_center.
            grad_centers_rows=model.center_loss.centers.grad[labs].numpy(),
            grad_centers_rows_idx=labs,
            grad_centers_abs_sum=float(model.center_loss.centers.grad.abs().sum()),
            grad_bn_weight=model.bn.weight.grad.numpy(),
            grad_fc_rows=model.fc_query.weight.grad[labs].numpy(),
            grad_fc_checksum=checksum(model.fc_query.weight.grad),
            bn_running_mean=model.bn.running_mean.numpy(),
            bn_running_var=model.bn.running_var.numpy(),
        )
        print(f"base_loss_{name}: total={float(out['loss']):.6f} parts={parts} "
              f"dist_ap={out['other']['step_dist_ap']:.4f} dist_an={out['other']['step_dist_an']:.4f}")


if __name__ == "__main__":
    generate()
