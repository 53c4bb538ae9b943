"""Drop-in for losses/triplet_loss.py of the reference: normalize, euclidean_dist,
cosine_dist, hard_example_mining, TripletLoss, CrossEntropyLabelSmooth -- same names,
arguments and return values, computed by the sm_90a kernels behind include/ctl_b200.h.
"""
from __future__ import annotations

import torch
from torch import nn

from .. import retrieval as _R
from ._fn import TripletFn, XentSmoothFn


def normalize(x, axis=-1):
    """losses/triplet_loss.py:16-24: x / (||x||_2 + 1e-12) along `axis`."""
    return 1.0 * x / (torch.norm(x, 2, axis, keepdim=True).expand_as(x) + 1e-12)


def euclidean_dist(x, y):
    """losses/triplet_loss.py:27-41: sqrt(clamp(|x|^2 + |y|^2 - 2 x.y, 1e-12)), [m, n].
    Forward value only (TripletLoss carries its own fused backward)."""
    return _R.dist_matrix(x, y, "euclidean_sqrt")


def cosine_dist(x: torch.Tensor, y: torch.Tensor, eps: float = 1e-12) -> torch.Tensor:
    """losses/triplet_loss.py:58-65: clamp(|1 - cos|, eps)."""
    if eps != 1e-12:
        raise NotImplementedError("the cosine kernel is built for the reference's eps=1e-12")
    return _R.dist_matrix(x, y, "cosine")


def hard_example_mining(dist_mat, labels, return_inds=False):
    """losses/triplet_loss.py:68-119: hardest positive (max, self included) and hardest
    negative (min) per anchor.  Index bookkeeping on an already materialised [N, N] matrix:
    thin torch glue -- the training path never materialises the matrix (TripletLoss below)."""
    assert len(dist_mat.size()) == 2
    assert dist_mat.size(0) == dist_mat.size(1)
    same = labels[:, None] == labels[None, :]
    dist_ap, p_inds = torch.where(same, dist_mat, dist_mat.new_full((), -float("inf"))).max(1)
    dist_an, n_inds = torch.where(~same, dist_mat, dist_mat.new_full((), float("inf"))).min(1)
    if return_inds:
        return dist_ap, dist_an, p_inds, n_inds
    return dist_ap, dist_an


class TripletLoss(object):
    """losses/triplet_loss.py:122-173.  Batch-hard triplet loss; forward + backward fused in
    ctl_triplet_step (Gram matrix, mining, hinge, and dE = rowsum(C) E - C E)."""

    def __init__(self, margin=None, dist_func="euclidean"):
        self.margin = margin  # None -> nn.SoftMarginLoss on (dist_an - dist_ap), triplet_loss.py:130-131
        self.dist_func_name = dist_func
        if dist_func == "cosine":
            self.dist_func = cosine_dist
        elif dist_func == "euclidean":
            self.dist_func = euclidean_dist
        else:
            raise KeyError(dist_func)

    def __call__(self, global_feat, labels, warmup_margin=False, print_data=False, normalize_feature=False,
                 mask=None):
        if normalize_feature:
            global_feat = normalize(global_feat, axis=-1)
        loss, dist_ap, dist_an = TripletFn.apply(global_feat, labels, mask, self.margin, self.margin is None,
                                                 self.dist_func_name == "cosine")
        if mask is not None:
            dist_ap, dist_an = dist_ap[mask], dist_an[mask]
        if print_data:
            print(f"LOSS: {loss.item()}")
            print(f"precision: {(dist_an > dist_ap).float().mean()}")
            print(f"proportion of triplets that satisfy margin: {(dist_an > dist_ap + (self.margin or 0.0)).float().mean()}")
            print(f"AP mean distance: {dist_ap.mean()}")
            print(f"AN mean distance: {dist_an.mean()}")
        return loss, dist_ap, dist_an


class CrossEntropyLabelSmooth(nn.Module):
    """losses/triplet_loss.py:176-205: y = (1 - eps) * onehot + eps / K;
    loss = (-y * log_softmax(inputs)).mean(0).sum()."""

    def __init__(self, num_classes, epsilon=0.1, use_gpu=True):
        super().__init__()
        self.num_classes = num_classes
        self.epsilon = epsilon
        self.use_gpu = use_gpu

    def forward(self, inputs, targets):
        if inputs.shape[1] != self.num_classes:
            raise ValueError(f"expected {self.num_classes} classes, got {inputs.shape[1]}")
        return XentSmoothFn.apply(inputs, targets, self.epsilon)
