"""Drop-in for utils/reid_metric.py of the reference (get_euclidean, get_cosine,
get_dist_func, R1_mAP) on the H100 distance kernel.

The distance functions return the full [m, n] matrix like the reference (on the device of
the inputs; host inputs are staged through the GPU and returned on the host).  R1_mAP.compute
does not build the matrix: normalisation, distances, ranking and CMC / mAP are fused into the
streamed evaluation (retrieval.evaluate_streamed).
"""
from __future__ import annotations

import os

import numpy as np
import torch

from .. import retrieval as _R
from .eval_reid import eval_func  # noqa: F401  (re-exported like the reference, reid_metric.py:20)


def _stage(t):
    t = torch.as_tensor(t)
    return (t if t.is_cuda else t.cuda(non_blocking=True)), t.device


def get_euclidean(x, y, **kwargs):
    """utils/reid_metric.py:25-33: SQUARED L2, |x|^2 + |y|^2 - 2 x.y (no clamp, no sqrt)."""
    xd, dev = _stage(x)
    yd, _ = _stage(y)
    out = _R.dist_matrix(xd, yd, "euclidean")
    return out if dev.type == "cuda" else out.to(dev)


def get_cosine(x: torch.Tensor, y: torch.Tensor, eps: float = 1e-12) -> torch.Tensor:
    """utils/reid_metric.py:51-59: clamp(|1 - cos(x, y)|, eps)."""
    if eps != 1e-12:
        raise NotImplementedError("the cosine kernel is built for the reference's eps=1e-12")
    xd, dev = _stage(x)
    yd, _ = _stage(y)
    out = _R.dist_matrix(xd, yd, "cosine")
    return out if dev.type == "cuda" else out.to(dev)


def get_dist_func(func_name="euclidean"):
    """utils/reid_metric.py:62-68 (an unknown name raises, as the reference's UnboundLocalError)."""
    if func_name == "cosine":
        dist_func = get_cosine
    elif func_name == "euclidean":
        dist_func = get_euclidean
    else:
        raise UnboundLocalError(f"unknown distance function {func_name!r}")
    print(f"Using {func_name} as distance function during evaluation")
    return dist_func


class R1_mAP:
    """utils/reid_metric.py:71-150.  Same constructor and `compute` signature."""

    def __init__(self, pl_module, num_query, max_rank=50, feat_norm=True):
        self.num_query = num_query
        self.max_rank = max_rank
        self.feat_norm = feat_norm
        self.pl_module = pl_module
        trainer = getattr(pl_module, "trainer", None)
        self.current_epoch = getattr(trainer, "current_epoch", 0)
        self.hparms = pl_module.hparams
        self.dist_name = self.hparms.SOLVER.DISTANCE_FUNC
        self.dist_func = get_dist_func(self.dist_name)
        self.dataset = None
        if getattr(self.hparms.TEST, "VISUALIZE", "no") == "yes":
            self.dataset = _eval_samples(trainer)

    def compute(self, feats, pids, camids, respect_camids=False):
        if self.feat_norm:
            print("The test feature is normalized")
        feats, _ = _stage(torch.as_tensor(feats).float())
        nq = self.num_query
        q_pids = np.asarray(pids[:nq])
        g_pids = np.asarray(pids[nq:])
        q_camids, g_camids = camids[:nq], camids[nq:]
        # reid_metric.py:113-136: F.normalize -> dist -> argsort -> eval_func(.., 50, ..), fused.
        # (the reference hard-codes max_rank=50 in the eval_func call, :134-136)
        # both operands are stored in identity order: the collect pass then skips every tile that cannot hold a positive
        # (retrieval.pid_order); results come back in the caller's indexing, bit-identical to the unsorted run
        qo = _R.pid_order(q_pids)
        go = _R.pid_order(g_pids) if len(g_pids) == feats.shape[0] - nq else None
        qp = _R.build_planes(feats[:nq], self.dist_name, self.feat_norm, order=qo)
        gp = _R.build_planes(feats[nq:], self.dist_name, self.feat_norm, order=go)
        res = _R.evaluate_streamed(qp, gp, q_pids, g_pids, q_camids, g_camids, 50, respect_camids)
        self.last_result = res
        hp = self.hparms
        if getattr(hp.TEST, "VISUALIZE", "no") == "yes":  # reid_metric.py:138-149, from the planes: no distmat
            from .visrank import visualize_ranked_planes

            print("Start visualization...")
            visualize_ranked_planes(qp, gp, self.dataset, hp, width=hp.INPUT.SIZE_TEST[1], height=hp.INPUT.SIZE_TEST[0],
                                    save_dir=os.path.join(hp.OUTPUT_DIR, "visrank"), topk=hp.TEST.VISUALIZE_TOPK)
        return res.cmc, res.mAP, res.all_topk


def _eval_samples(trainer):
    """reid_metric.py:87-90: the (path, pid, camid, index) samples of the validation (else the test) loader, which
    TEST.VISUALIZE needs for the image files."""
    for attr in ("val_dataloaders", "test_dataloaders"):
        try:
            return getattr(trainer, attr)[0].dataset.samples
        except (AttributeError, IndexError, KeyError, TypeError):
            continue
    raise ValueError("TEST.VISUALIZE = 'yes' needs the image paths: pl_module.trainer.val_dataloaders[0] (or "
                     "test_dataloaders[0]) must have a dataset with `samples`")
