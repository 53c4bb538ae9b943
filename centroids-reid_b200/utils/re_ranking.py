"""k-reciprocal re-ranking (Zhong, Zheng, Cao, Li, "Re-ranking Person Re-identification with k-reciprocal Encoding",
CVPR 2017) under the name and signature of the reid-strong-baseline lineage that utils/reid_metric.py credits, computed
on the H100 (retrieval.rerank; semantics in include/ctl_b200.h)."""
from __future__ import annotations

import numpy as np
import torch

from .. import retrieval as _R


def re_ranking(probFea, galFea, k1, k2, lambda_value, local_distmat=None, only_local=False):
    """Re-ranked [Q, G] distances of query features `probFea` [Q, d] against gallery features `galFea` [G, d], as a numpy
    float32 array.  Host tensors are staged to the current CUDA device.  V and the Jaccard sums are float32 (the lineage's
    float16 storage is not reproduced) and equal distances are ordered by index.  AlignedReID local distances
    (`local_distmat`, `only_local`) are not part of this model."""
    if local_distmat is not None or only_local:
        raise NotImplementedError("local_distmat / only_local (AlignedReID local features) are not supported")
    q = torch.as_tensor(probFea)
    g = torch.as_tensor(galFea)
    if not q.is_cuda:
        q = q.cuda(non_blocking=True)
    if not g.is_cuda:
        g = g.to(q.device, non_blocking=True)
    return _R.rerank(q, g, int(k1), int(k2), float(lambda_value)).cpu().numpy().astype(np.float32, copy=False)
