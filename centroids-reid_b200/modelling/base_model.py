"""Drop-in for train_base_model.CTLModel, the paper's baseline: the CTL model's trunk, head and losses without the
centroid rounds (train_base_model.py:27-96).

BaseModel inherits everything but the loss from CTLModel (modelling/ctl_model.py): the constructor
(modelling/bases.py:53-90), evaluation, `configure_optimizers` and `optimizer_step_manual` (warm-up LR rule, loss
scaler, center-gradient rescale by 1 / CENTER_LOSS_WEIGHT, `opt_center.step()`, invalidating the packed eval weights).
Its loss is one fused, host-sync-free kernel enqueue (ctl_base_loss_step, include/ctl_b200.h) that differs from the CTL
step in its row sets: the center loss and the BatchNorm1d -> fc_query -> label-smoothed CE head see ALL B rows, mock
rows included, and only the query triplet's anchors are masked to `isReal`.
"""
from __future__ import annotations

from .. import _native as N
from ..losses._fn import BaseStepFn
from .ctl_model import CTLModel, fused_step_done

BASE_LOSS_NAMES = ("total", "query_xent", "query_triplet", "query_center", "step_dist_ap", "step_dist_an")


def base_losses(module, features, class_labels, is_real):
    """train_base_model.py:60-75 in one call: returns (total_loss tensor with autograd into features / centers /
    bn.weight / fc_query.weight, parts float32[6] on the device in BASE_LOSS_NAMES order).  Every TripletLoss variant
    (SOLVER.DISTANCE_FUNC euclidean / cosine, SOLVER.MARGIN None -> SoftMarginLoss) runs fused; no host synchronisation
    after the first step."""
    S = module.hparams.SOLVER
    if S.DISTANCE_FUNC not in ("euclidean", "cosine"):
        raise ValueError(f"SOLVER.DISTANCE_FUNC={S.DISTANCE_FUNC!r}: TripletLoss knows 'euclidean' and 'cosine' "
                         "(losses/triplet_loss.py:133-136)")
    if not module.bn.training:
        raise NotImplementedError("the fused loss step normalises with BATCH statistics (nn.BatchNorm1d in train mode, as in "
                                  "the reference's training_step); call module.train() / module.bn.train() first")
    B, D = features.shape
    soft = S.MARGIN is None
    cfg = N.BaseLossConfig(B, D, module.fc_query.weight.shape[0], 0.0 if soft else float(S.MARGIN), int(soft),
                           int(S.DISTANCE_FUNC == "cosine"), float(S.CENTER_LOSS_WEIGHT), float(S.QUERY_XENT_WEIGHT),
                           float(S.QUERY_CONTRASTIVE_WEIGHT), float(module.bn.eps), float(module.bn.momentum), 0.1)
    total, parts = BaseStepFn.apply(features, module.center_loss.centers, module.bn.weight, module.fc_query.weight,
                                    module.bn.bias, module.bn.running_mean, module.bn.running_var, class_labels, is_real,
                                    cfg)
    # a label outside [0, num_classes) comes back as a NaN with a payload (the centers are indexed by label)
    fused_step_done(module, parts, "base-model training step")
    return total, parts


class BaseModel(CTLModel):
    """train_base_model.CTLModel (train_base_model.py:27-96) on the H100 engine.  `training_step` is CTLModel's
    (train_base_model.py:38-96 is train_ctl_model.py:38-179 with another loss): with optimizers attached it runs the whole
    manual-optimisation iteration and returns {"loss", "other": {step_dist_ap, step_dist_an}}; without, it returns
    {"loss" (differentiable), "parts"}."""

    def training_step_from_features(self, features, class_labels, is_real):
        """Everything of training_step after `_, features = self.backbone(x)` (train_base_model.py:57) up to and
        including the loss assembly (:75).  Returns {"loss" (differentiable), "parts" (BASE_LOSS_NAMES order)}."""
        total, parts = base_losses(self, features, class_labels, is_real)
        return {"loss": total, "parts": parts}

    def _log_step(self, total, parts):
        """train_base_model.py:84-96.  The reference zips FOUR loss names with THREE values, so `centroid_triplet` stays
        an empty list; dist_ap / dist_an are the means over the real anchors."""
        for name, val in zip(self.losses_names, (parts[1], parts[2], parts[3])):
            self.losses_dict[name].append(val)
        return {"loss": total.detach(), "other": {"step_dist_ap": parts[4], "step_dist_an": parts[5]}}
