"""TEST INFRASTRUCTURE ONLY -- CPU oracle for the centroid-triplet re-ID hot path.

A CPU restatement (torch-CPU fp32 for the differentiable parts, numpy for ranks / CMC / mAP)
of the algorithms on the path named by BASELINE.json:north_star.  Each function cites the
reference file:line it follows (paths relative to /root/reference, commit a1825b7).

Pinning: the reference ships no tests and no golden vectors (SURVEY.md section 4), so this
restatement is pinned against outputs of the *reference itself*, executed in the build
container through ``oracle/ref_import.py`` by ``oracle/make_golden.py``; the resulting
vectors are committed under ``tests/golden/`` and checked by ``tests/test_oracle_golden.py``
(CPU, ``-m "not gpu"``), and -- when /root/reference is mounted -- directly against the
live reference by ``tests/test_oracle_golden.py``.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl
reference`` legs may import this module.  The product (``centroids-reid_b200``) never does.
"""
from __future__ import annotations

import math
from collections import OrderedDict, defaultdict

import numpy as np
import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------
# distances  (losses/triplet_loss.py:27-65, utils/reid_metric.py:25-59)
# --------------------------------------------------------------------------------------


def _f(x: torch.Tensor) -> torch.Tensor:
    """The reference's `.float()` casts (triplet_loss.py:39, center_loss.py:37).  float64 inputs
    are left alone so the same restatement can serve as a higher-precision checker."""
    return x if x.dtype == torch.float64 else x.float()


def euclidean_dist(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """losses/triplet_loss.py:27-41 -- sqrt(clamp(|x|^2 + |y|^2 - 2 x.y, 1e-12)), fp32."""
    xx = (x * x).sum(1, keepdim=True)
    yy = (y * y).sum(1, keepdim=True).t()
    d = torch.addmm(xx + yy, _f(x), _f(y).t(), beta=1.0, alpha=-2.0)
    return d.clamp(min=1e-12).sqrt()


def cosine_similarity(x, y, eps=1e-12):
    """losses/triplet_loss.py:44-55 == utils/reid_metric.py:36-48."""
    xn = x.norm(dim=1)[:, None]
    yn = y.norm(dim=1)[:, None]
    return (x / torch.clamp(xn, min=eps)) @ (y / torch.clamp(yn, min=eps)).t()


def cosine_dist(x, y, eps=1e-12):
    """losses/triplet_loss.py:58-65 == utils/reid_metric.py:51-59: clamp(|1 - cos|, eps)."""
    return (1.0 - cosine_similarity(x, y, eps)).abs().clamp(min=eps)


def get_euclidean(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """utils/reid_metric.py:25-33 -- SQUARED L2, no clamp, no sqrt."""
    xx = (x * x).sum(1, keepdim=True)
    yy = (y * y).sum(1, keepdim=True).t()
    return torch.addmm(xx + yy, x, y.t(), beta=1.0, alpha=-2.0)


get_cosine = cosine_dist


def get_dist_func(name="euclidean"):
    """utils/reid_metric.py:62-68."""
    return {"euclidean": get_euclidean, "cosine": get_cosine}[name]


# --------------------------------------------------------------------------------------
# batch-hard triplet  (losses/triplet_loss.py:68-173)
# --------------------------------------------------------------------------------------


def hard_example_mining(dist_mat: torch.Tensor, labels: torch.Tensor):
    """losses/triplet_loss.py:68-119.  Per anchor: max over same-label columns (self
    included), min over different-label columns.  The reference's boolean-index + view
    requires equally many positives per anchor; the masked max/min below is the same
    function on every input the reference accepts."""
    same = labels[:, None] == labels[None, :]
    neg_inf = torch.full_like(dist_mat, -float("inf"))
    pos_inf = torch.full_like(dist_mat, float("inf"))
    dist_ap = torch.where(same, dist_mat, neg_inf).max(dim=1).values
    dist_an = torch.where(~same, dist_mat, pos_inf).min(dim=1).values
    return dist_ap, dist_an


def triplet_loss(feat, labels, margin=0.5, mask=None, dist_func="euclidean"):
    """TripletLoss.__call__, losses/triplet_loss.py:139-173 (MarginRankingLoss, y=1, or
    SoftMarginLoss when margin is None).  Returns (loss, dist_ap, dist_an)."""
    d = euclidean_dist(feat, feat) if dist_func == "euclidean" else cosine_dist(feat, feat)
    ap, an = hard_example_mining(d, labels)
    if mask is not None:
        ap, an = ap[mask], an[mask]
    if margin is not None:
        loss = torch.clamp(ap - an + margin, min=0).mean()
    else:
        loss = F.softplus(-(an - ap)).mean()
    return loss, ap, an


# --------------------------------------------------------------------------------------
# center loss / label-smoothed CE / head  (losses/center_loss.py:26-45,
# losses/triplet_loss.py:194-205, modelling/bases.py:83-87)
# --------------------------------------------------------------------------------------


def center_loss(x, labels, centers):
    """losses/center_loss.py:26-45.  The full [B,C] matrix is masked by the one-hot labels
    and clamped element-wise, so each of the B*(C-1) masked zeros contributes 1e-12."""
    b, c = x.shape[0], centers.shape[0]
    xx = (x * x).sum(1, keepdim=True)
    cc = (centers * centers).sum(1, keepdim=True).t()
    distmat = torch.addmm(xx + cc, _f(x), centers.t(), beta=1.0, alpha=-2.0)
    onehot = F.one_hot(labels, c).to(distmat.dtype)
    return (distmat * onehot).clamp(min=1e-12, max=1e12).sum() / b


def cross_entropy_label_smooth(logits, targets, num_classes, epsilon=0.1):
    """losses/triplet_loss.py:194-205: (-t * log_softmax).mean(0).sum()."""
    logp = F.log_softmax(logits, dim=1)
    t = F.one_hot(targets, num_classes).to(logp.dtype)
    t = (1 - epsilon) * t + epsilon / num_classes
    return (-t * logp).mean(0).sum()


# --------------------------------------------------------------------------------------
# CTL training-step losses  (train_ctl_model.py:54-152, modelling/bases.py:359-384)
# --------------------------------------------------------------------------------------


def create_masks_train(class_labels: np.ndarray):
    """modelling/bases.py:359-384, restated.  masks[r, idx] is False for the r-th member of
    every pid (the round-r query) and True elsewhere ("True for gallery"); once a pid has
    run out of members its whole block is False.  Returns (masks[max_k, B] bool,
    labels_list).  NB (reference quirk kept): for the FIRST pid (i == 0) an exhausted list
    indexes lens_list_cs[-1], i.e. zeroes a slice starting at B -> a no-op."""
    labels = np.asarray(class_labels)
    groups: "OrderedDict[int, list]" = OrderedDict()
    for idx, pid in enumerate(labels.tolist()):
        groups.setdefault(pid, []).append(idx)
    labels_list = [list(v) for v in groups.values()]
    lens = [len(v) for v in labels_list]
    cs = np.cumsum(lens)
    max_k = max(lens)
    masks = np.ones((max_k, len(labels)), dtype=bool)
    for r in range(max_k):
        for i, members in enumerate(labels_list):
            if r < len(members):
                masks[r, members[r]] = False
            else:
                start = cs[i - 1]
                masks[r, start : start + lens[i]] = False
    return masks, labels_list


def ctl_step_losses(
    feats: torch.Tensor,
    labels: torch.Tensor,
    is_real: torch.Tensor,
    num_instance: int,
    centers: torch.Tensor,
    bn_weight: torch.Tensor,
    bn_bias: torch.Tensor,
    fc_weight: torch.Tensor,
    *,
    margin=0.5,
    center_loss_weight=5e-4,
    query_xent_weight=1.0,
    query_contrastive_weight=1.0,
    centroid_contrastive_weight=1.0,
    bn_eps=1e-5,
    epsilon=0.1,
    dist_func="euclidean",
):
    """Everything CTLModel.training_step computes after the trunk and before backward
    (train_ctl_model.py:54-152) as a differentiable torch-CPU function of
    (feats, centers, bn_weight, fc_weight).

    Returns dict(total, xent, triplet, center, ctl, dist_ap, dist_an, l2_centroid).
    """
    K = num_instance
    B, D = feats.shape
    # train_ctl_model.py:56 -- number of distinct pids; batch is pid-major blocks of K (A0)
    P = len(np.unique(labels.detach().cpu().numpy()))
    assert P * K == B, "batch contract: P pids x K instances, pid-major (datasets/bases.py:346-406)"

    # :62-67 image-level batch-hard triplet, anchors restricted to real rows
    l_q, _, _ = triplet_loss(feats, labels, margin, mask=is_real, dist_func=dist_func)
    l_q = l_q * query_contrastive_weight

    # :69-77 center loss + BN1d(train) + bias-free fc + label-smoothed CE on real rows only
    lab_r = labels[is_real]
    f_r = feats[is_real]
    l_cen = center_loss_weight * center_loss(f_r, lab_r, centers)
    bn_f = F.batch_norm(f_r, None, None, bn_weight, bn_bias, True, 0.1, bn_eps)
    logits = bn_f @ fc_weight.t()
    l_x = cross_entropy_label_smooth(logits, lab_r, fc_weight.shape[0], epsilon) * query_xent_weight

    # :79-104 masks and per-round centroids.  Closed form (probe-verified in SURVEY A.1):
    #   M_r[c, s] = (s != r) & R[c, r] & R[c, s],  R = is_real.view(P, K)
    R = is_real.view(P, K)
    masks_np, _ = create_masks_train(labels.detach().cpu().numpy())
    masks = torch.from_numpy(masks_np)
    t_re = R[:, :, None].expand(P, K, K).permute(1, 0, 2).reshape(K, P * K) & is_real[None, :]
    masks = masks & t_re
    mf = masks.to(feats.dtype)
    padded = mf[:, :, None] * feats[None]  # [K, B, D]
    cm = masks.view(K, P, K)
    valid = cm.sum(-1)
    cent = padded.view(K, P, K, D).sum(-2) / valid.masked_fill(valid == 0, 1)[..., None].to(feats.dtype)

    losses, aps, ans, l2s = [], [], [], []
    for r in range(K):  # :112-140
        if int((valid[r] > 0).sum()) <= 1:
            continue
        sel = (~masks[r]) & t_re[r]
        q = feats[sel]
        ql = labels[sel]
        c = cent[r]
        c = c[c.abs().sum(1) > 1e-7]
        emb = torch.cat((q, c))
        lab = torch.cat((ql, ql))
        l, ap, an = triplet_loss(emb, lab, margin, dist_func=dist_func)
        losses.append(l)
        aps.append(ap.detach().mean())
        ans.append(an.detach().mean())
        l2s.append(c.norm(dim=1).mean())
    l_ctl = torch.stack(losses).mean() * centroid_contrastive_weight  # :142-145
    total = l_ctl + l_cen + l_x + l_q  # :150-152
    return dict(
        total=total,
        xent=l_x,
        triplet=l_q,
        center=l_cen,
        ctl=l_ctl,
        dist_ap=torch.stack(aps).mean(),
        dist_an=torch.stack(ans).mean(),
        l2_centroid=torch.stack(l2s).mean().detach(),
    )


# --------------------------------------------------------------------------------------
# centroids  (modelling/bases.py:92-95,179-262, inference/inference_utils.py:147-159)
# --------------------------------------------------------------------------------------


def calculate_centroids_by_pid(embeddings: np.ndarray, pid_path_index: dict):
    """inference/inference_utils.py:147-159: mean of the rows of every pid, in dict order."""
    pids, cents = [], []
    for pid, idx in pid_path_index.items():
        cents.append(np.asarray(embeddings)[idx].sum(0) / len(idx))
        pids.append(pid)
    return np.stack(cents), np.array(pids, dtype=np.str_)


def validation_create_centroids(embeddings, labels, camids, num_query, respect_camids=False):
    """modelling/bases.py:179-262.  Gallery rows collapse to one centroid per pid, or (with
    respect_camids) one per distinct set of 'other-camera' gallery images per query camid.
    NB reference quirk kept: `camids[inds]` (:214) indexes the FULL camid array with
    gallery-relative indices."""
    embeddings = torch.as_tensor(embeddings)
    labels = np.asarray(labels)
    camids = np.asarray(camids)
    emb_q = embeddings[:num_query]
    lab_q = labels[:num_query]
    emb_g = embeddings[num_query:]
    lab_g = labels[num_query:]
    l2i, l2i_q = defaultdict(list), defaultdict(list)
    for i, l in enumerate(lab_g.tolist()):
        l2i[l].append(i)
    for i, l in enumerate(lab_q.tolist()):
        l2i_q[l].append(i)
    cent_emb, cent_lab, cent_cam = [], [], []
    for label in sorted(l2i.keys()):
        inds = l2i[label]
        if respect_camids:
            seen = set()
            cam_g = camids[inds]
            cam_q = camids[l2i_q[label]]
            for cur in sorted(np.unique(cam_q).tolist()):
                sel = np.where(cam_g != cur)[0]
                if sel.shape[0] == 0:
                    continue
                used = tuple(sorted(np.unique([c for c in cam_g.tolist() if c != cur]).tolist()))
                if used not in seen:
                    seen.add(used)
                    rows = emb_g[inds][sel]
                    cent_emb.append(rows.sum(0) / rows.shape[0])
                    cent_cam.append(list(used))
                    cent_lab.append(label)
        else:
            rows = emb_g[inds]
            cent_lab.append(label)
            cent_emb.append(rows.sum(0) / rows.shape[0])
    out_emb = torch.cat((emb_q, torch.stack(cent_emb)), 0)
    out_lab = np.hstack((lab_q, np.asarray(cent_lab)))
    if respect_camids:
        out_cam = [[c] for c in camids[:num_query].tolist()] + cent_cam
    else:
        # reference quirk kept (bases.py:255-260): the ones are sized from the ALREADY
        # concatenated label array, so the dummy camid vector is num_query entries too long;
        # harmless downstream because eval_func only indexes its first n_gallery entries.
        out_cam = np.hstack((np.zeros_like(lab_q), np.ones_like(out_lab)))
    return out_emb, out_lab, out_cam


# --------------------------------------------------------------------------------------
# ranks / CMC / mAP  (utils/reid_metric.py:112-136, utils/eval_reid.py:25-92)
# --------------------------------------------------------------------------------------

K_LIST = (1, 5, 10, 20, 50)


def rank_indices(distmat: np.ndarray) -> np.ndarray:
    """utils/reid_metric.py:129,132 `np.argsort(distmat, axis=1)` made canonical: the
    reference's default (unstable) sort leaves tie order unspecified; the contract of this
    repo is ascending (distance, gallery index), i.e. kind='stable'."""
    return np.argsort(np.asarray(distmat), axis=1, kind="stable")


def _junk_matrix(q_pids, g_pids, q_camids, g_camids, respect_camids):
    """utils/eval_reid.py:52-59."""
    same_pid = g_pids[None, :] == q_pids[:, None]
    if respect_camids:
        in_set = np.zeros((len(q_pids), len(g_pids)), dtype=bool)
        for j, cams in enumerate(g_camids):
            cams = set(np.atleast_1d(cams).tolist())
            for i, qc in enumerate(q_camids):
                qv = qc[0] if isinstance(qc, (list, tuple, np.ndarray)) else qc
                in_set[i, j] = qv in cams
        return same_pid & in_set
    # g_camids may be longer than the gallery (validation_create_centroids quirk); the
    # reference only ever indexes it with gallery positions (eval_reid.py:57)
    g_cam = np.asarray(g_camids)[: len(g_pids)]
    return same_pid & (g_cam[None, :] == np.asarray(q_camids)[:, None])


def eval_func(indices, q_pids, g_pids, q_camids, g_camids, max_rank=50, respect_camids=False):
    """utils/eval_reid.py:25-92, per query (junk removal, CMC, AP over the full kept
    ranking, top-k hits).  Restated per-query with numpy; float64 throughout like the
    reference's python floats.  Returns (all_cmc f32[max_rank], mAP, all_topk[5],
    single_performance[nq,3])."""
    indices = np.asarray(indices)
    q_pids, g_pids = np.asarray(q_pids), np.asarray(g_pids)
    num_q, num_g = indices.shape
    max_rank = min(max_rank, num_g)
    junk_all = _junk_matrix(q_pids, g_pids, q_camids, g_camids, respect_camids)
    all_cmc, all_ap, topk, single = [], [], [], []
    for q in range(num_q):
        order = indices[q]
        keep = ~junk_all[q][order]
        hits = (g_pids[order] == q_pids[q])[keep].astype(np.int32)
        if not hits.any():
            continue
        c = hits.cumsum()
        cmc = np.minimum(c, 1)[:max_rank]
        if cmc.shape[0] < max_rank:  # reference would build a ragged array and raise (A.4)
            cmc = np.concatenate([cmc, np.full(max_rank - cmc.shape[0], cmc[-1])])
        all_cmc.append(cmc)
        prec = c / (np.arange(len(c)) + 1.0)
        ap = float((prec * hits).sum() / hits.sum())
        all_ap.append(ap)
        single.append([q, q_pids[q], ap])
        topk.append([int(hits[:k].any()) for k in K_LIST])
    all_cmc = np.asarray(all_cmc).astype(np.float32).sum(0) / float(len(all_ap))
    return all_cmc, float(np.mean(all_ap)), np.mean(np.vstack(topk), 0), np.array(single)


def r1_map_compute(feats, pids, camids, num_query, feat_norm=True, dist="euclidean", respect_camids=False):
    """R1_mAP.compute, utils/reid_metric.py:112-136 (visualisation excluded)."""
    feats = torch.as_tensor(feats).float()
    if feat_norm:
        feats = F.normalize(feats, dim=1, p=2)
    qf, gf = feats[:num_query], feats[num_query:]
    q_pids, g_pids = np.asarray(pids[:num_query]), np.asarray(pids[num_query:])
    q_cam, g_cam = camids[:num_query], camids[num_query:]
    distmat = get_dist_func(dist)(qf, gf).numpy()
    idx = rank_indices(distmat)
    cmc, mAP, all_topk, _ = eval_func(idx, q_pids, g_pids, q_cam, g_cam, 50, respect_camids)
    return cmc, mAP, all_topk


def topk_similar(qf, gf, topk=100, dist="euclidean", normalize=False):
    """inference/get_similar.py:104-128: optional normalise, dist, argsort, [:, :topk],
    gathered distances."""
    qf, gf = torch.as_tensor(qf).float(), torch.as_tensor(gf).float()
    if normalize:
        qf, gf = F.normalize(qf, dim=1, p=2), F.normalize(gf, dim=1, p=2)
    d = get_dist_func(dist)(qf, gf).numpy()
    idx = rank_indices(d)[:, :topk]
    return idx, np.take_along_axis(d, idx, axis=1)


# --------------------------------------------------------------------------------------
# trunk  (modelling/backbones/resnet.py:51-133, resnet_ibn_a.py:18-141, baseline.py:91-96,
#         modelling/bases.py:169-177)
# --------------------------------------------------------------------------------------

R50_LAYERS = (3, 4, 6, 3)


def make_trunk_state(seed=0, ibn=False, num_classes=None, layers=R50_LAYERS, randomize_bn=True):
    """Deterministic synthetic weights with the reference's state_dict keys/shapes
    (`base.*` = modelling/backbones/resnet.py:90-120 / resnet_ibn_a.py:77-124).  Conv weights
    ~ N(0, sqrt(2/(k*k*Cout))) (resnet.py:156-164 random_init), BN affine and running
    statistics randomised so that folding is exercised (SURVEY 8d)."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()

    def conv(name, cout, cin, k):
        sd[name + ".weight"] = torch.randn(cout, cin, k, k, generator=g) * math.sqrt(2.0 / (k * k * cout))

    def bn(name, c):
        if randomize_bn:
            # residual-branch BNs (bn3) get a small gain, as in trained nets, so that the
            # 16-block residual sum stays O(1) and an fp16 trunk is well inside its range
            gain = 0.25 if name.endswith("bn3") else 1.0
            sd[name + ".weight"] = gain * (0.5 + torch.rand(c, generator=g))
            sd[name + ".bias"] = 0.1 * torch.randn(c, generator=g)
            sd[name + ".running_mean"] = 0.1 * torch.randn(c, generator=g)
            sd[name + ".running_var"] = 0.5 + torch.rand(c, generator=g)
        else:
            sd[name + ".weight"] = torch.ones(c)
            sd[name + ".bias"] = torch.zeros(c)
            sd[name + ".running_mean"] = torch.zeros(c)
            sd[name + ".running_var"] = torch.ones(c)
        sd[name + ".num_batches_tracked"] = torch.zeros((), dtype=torch.long)

    def inorm(name, c):
        sd[name + ".weight"] = 0.5 + torch.rand(c, generator=g) if randomize_bn else torch.ones(c)
        sd[name + ".bias"] = 0.1 * torch.randn(c, generator=g) if randomize_bn else torch.zeros(c)

    conv("conv1", 64, 3, 7)
    bn("bn1", 64)
    inplanes = 64
    for li, (planes, nblk) in enumerate(zip((64, 128, 256, 512), layers), start=1):
        for b in range(nblk):
            p = f"layer{li}.{b}"
            conv(p + ".conv1", planes, inplanes, 1)
            if ibn and planes != 512:  # resnet_ibn_a.py:116-119
                half = planes // 2
                inorm(p + ".bn1.IN", half)
                bn(p + ".bn1.BN", planes - half)
            else:
                bn(p + ".bn1", planes)
            conv(p + ".conv2", planes, planes, 3)
            bn(p + ".bn2", planes)
            conv(p + ".conv3", planes * 4, planes, 1)
            bn(p + ".bn3", planes * 4)
            if b == 0:
                conv(p + ".downsample.0", planes * 4, inplanes, 1)
                bn(p + ".downsample.1", planes * 4)
                inplanes = planes * 4
    if ibn:  # unused fc carried by ResNet_IBN (resnet_ibn_a.py:92-93)
        sd["fc.weight"] = torch.zeros(1000, 2048)
        sd["fc.bias"] = torch.zeros(1000)
    return sd


def _bn(x, sd, name, train, eps=1e-5):
    return F.batch_norm(
        x, sd[name + ".running_mean"].clone(), sd[name + ".running_var"].clone(),
        sd[name + ".weight"], sd[name + ".bias"], train, 0.1, eps,
    )


def _norm1(x, sd, p, ibn_block, train):
    """bn1 of a bottleneck: plain BN, or IBN (resnet_ibn_a.py:18-32): InstanceNorm(affine,
    instance statistics also in eval) on the first half of the channels, BN on the rest."""
    if not ibn_block:
        return _bn(x, sd, p + ".bn1", train)
    half = sd[p + ".bn1.IN.weight"].shape[0]
    a = F.instance_norm(x[:, :half].float().contiguous(), None, None,
                        sd[p + ".bn1.IN.weight"], sd[p + ".bn1.IN.bias"], True, 0.1, 1e-5)
    b = _bn(x[:, half:].contiguous(), sd, p + ".bn1.BN", train)
    return torch.cat((a, b), 1)


def trunk_forward(x, sd, last_stride=1, ibn=False, train=False, layers=R50_LAYERS):
    """ResNet.forward (resnet.py:122-133; NO ReLU after the stem) / ResNet_IBN.forward
    (resnet_ibn_a.py:126-141; stem HAS ReLU) -> base_out [B,2048,H/16,W/16] at last_stride 1."""
    x = F.conv2d(x, sd["conv1.weight"], None, 2, 3)
    x = _bn(x, sd, "bn1", train)
    if ibn:
        x = F.relu(x)
    x = F.max_pool2d(x, 3, 2, 1)
    for li, (planes, nblk) in enumerate(zip((64, 128, 256, 512), layers), start=1):
        stride0 = 1 if li == 1 else (last_stride if li == 4 else 2)
        for b in range(nblk):
            p = f"layer{li}.{b}"
            stride = stride0 if b == 0 else 1
            out = F.conv2d(x, sd[p + ".conv1.weight"])
            out = F.relu(_norm1(out, sd, p, ibn and planes != 512, train))
            out = F.conv2d(out, sd[p + ".conv2.weight"], None, stride, 1)
            out = F.relu(_bn(out, sd, p + ".bn2", train))
            out = F.conv2d(out, sd[p + ".conv3.weight"])
            out = _bn(out, sd, p + ".bn3", train)
            if b == 0:
                res = F.conv2d(x, sd[p + ".downsample.0.weight"], None, stride)
                res = _bn(res, sd, p + ".downsample.1", train)
            else:
                res = x
            x = F.relu(out + res)
    return x


def baseline_forward(x, sd, **kw):
    """Baseline.forward, modelling/baseline.py:91-96 -> (base_out, global_feat[B,2048])."""
    base = trunk_forward(x, sd, **kw)
    return base, base.mean(dim=(2, 3))


def embed_forward(x, sd, bn_sd, **kw):
    """ModelBase.validation_step (modelling/bases.py:169-177) == inference_utils._inference
    (inference/inference_utils.py:104-113): eval trunk -> GAP -> eval BatchNorm1d."""
    _, gf = baseline_forward(x, sd, train=False, **kw)
    return F.batch_norm(gf, bn_sd["running_mean"], bn_sd["running_var"], bn_sd["weight"], bn_sd["bias"],
                        False, 0.1, 1e-5)


def trunk_forward_fp16sim(x, sd, last_stride=1, ibn=False, layers=R50_LAYERS):
    """Same-precision checker for the fp16 engine: trunk_forward(eval) with the rounding points
    of the H100 path made explicit -- eval BatchNorm folded into fp16 weights, fp32
    accumulation, every stored activation rounded to fp16 (the reference under AMP has the same
    class of rounding, SURVEY A.3; an fp16 trunk cannot meet 1e-4 against the fp32 reference, so
    parity of the trunk is defined against this function and reported against the fp32 one)."""
    eps = 1e-5

    def fold(wname, bnname, sl=slice(None)):
        sc = sd[bnname + ".weight"] / torch.sqrt(sd[bnname + ".running_var"] + eps)
        b = sd[bnname + ".bias"] - sd[bnname + ".running_mean"] * sc
        return sd[wname][sl] * sc[:, None, None, None], b

    def q(t):  # fp16 storage
        return t.half().float()

    w, b = fold("conv1.weight", "bn1")
    x = F.conv2d(q(x), q(w), b, 2, 3)  # tensor-core stem: fp16 input crop and weights, fp32 accumulate
    if ibn:
        x = F.relu(x)
    x = F.max_pool2d(q(x), 3, 2, 1)
    for li, (planes, nblk) in enumerate(zip((64, 128, 256, 512), layers), start=1):
        stride0 = 1 if li == 1 else (last_stride if li == 4 else 2)
        for bi in range(nblk):
            p = f"layer{li}.{bi}"
            stride = stride0 if bi == 0 else 1
            if ibn and planes != 512:
                half = planes // 2
                wb, bb = fold(p + ".conv1.weight", p + ".bn1.BN", slice(half, None))
                raw = q(F.conv2d(x, q(sd[p + ".conv1.weight"][:half])))
                a = F.instance_norm(raw, None, None, sd[p + ".bn1.IN.weight"], sd[p + ".bn1.IN.bias"], True, 0.1, eps)
                o1 = q(F.relu(torch.cat((a, F.conv2d(x, q(wb), bb)), 1)))
            else:
                w1, b1 = fold(p + ".conv1.weight", p + ".bn1")
                o1 = q(F.relu(F.conv2d(x, q(w1), b1)))
            w2, b2 = fold(p + ".conv2.weight", p + ".bn2")
            o2 = q(F.relu(F.conv2d(o1, q(w2), b2, stride, 1)))
            w3, b3 = fold(p + ".conv3.weight", p + ".bn3")
            if bi == 0:
                wd, bd = fold(p + ".downsample.0.weight", p + ".downsample.1")
                res = q(F.conv2d(x, q(wd), bd, stride))
            else:
                res = x
            x = q(F.relu(F.conv2d(o2, q(w3), b3) + res))
    return x, x.mean(dim=(2, 3))


class _RoundHalfSTE(torch.autograd.Function):
    """fp16 storage rounding in the forward, identity in the backward (the engine's backward is checked against
    the exact derivative of the rounded forward)."""

    @staticmethod
    def forward(ctx, t):
        return t.half().to(t.dtype)

    @staticmethod
    def backward(ctx, g):
        return g


def trunk_train_fp16sim(x, sd, dfeat=None, last_stride=1, layers=R50_LAYERS, momentum=0.1, forced=None, ibn=False,
                        round_fp16=True):
    """Train-mode trunk (ResNet.forward resnet.py:122-133 with BatchNorm2d batch statistics, Bottleneck.forward
    :67-87) in float64 with the H100 training path's rounding points: fp16 crops and conv weights, every stored
    activation (conv output, BN/ReLU output) rounded to fp16, statistics / BN arithmetic / GAP in full precision.
    Returns (global_feat, grads, running) where grads maps state_dict names -> d(sum(global_feat * dfeat))/d(param)
    and running holds the updated running statistics.  ibn=True: the IBN-a variant (resnet_ibn_a.py:18-32,54-74,126-141:
    ReLU after the stem; bn1 of layer1-3 = InstanceNorm2d(affine) on the first half of the channels, BatchNorm2d on
    the rest).

    `forced`: optional list of (y, z) NCHW tensors, one per conv+BN in execution order (stem, then per block conv1,
    conv2, [downsample], conv3): the VALUES of the stored activations are replaced by these (the engine's own fp16
    tensors) while the derivative still flows through this function's arithmetic.  ReLU masks are discontinuous,
    so two correct fp16 forwards that differ in the last bit produce visibly different gradients; teacher-forcing
    the stored activations isolates the backward arithmetic from that effect."""
    eps = 1e-5
    # round_fp16=False drops the engine's storage rounding: the function is then the reference's own train-mode
    # arithmetic in float64 (pinned against the reference run in fp32, tests/golden/trunk_train.npz)
    q = _RoundHalfSTE.apply if round_fp16 else (lambda t: t)
    P = {k: v.detach().double().requires_grad_(True) for k, v in sd.items()
         if v.is_floating_point() and "running" not in k}
    running = {}
    it = iter(forced) if forced is not None else None

    def force(t, val):
        return t if val is None else val.double() + (t - t.detach())

    def batch_norm(y, name):
        mean = y.mean(dim=(0, 2, 3))
        var = y.var(dim=(0, 2, 3), unbiased=False)
        cnt = y.numel() / y.shape[1]
        running[name + ".running_mean"] = (1 - momentum) * sd[name + ".running_mean"].double() + momentum * mean.detach()
        running[name + ".running_var"] = ((1 - momentum) * sd[name + ".running_var"].double()
                                          + momentum * var.detach() * cnt / max(cnt - 1, 1))
        return ((y - mean[None, :, None, None]) / torch.sqrt(var + eps)[None, :, None, None]
                * P[name + ".weight"][None, :, None, None] + P[name + ".bias"][None, :, None, None])

    def conv_bn(a, conv, name, k, stride, res=None, relu=True, ibn_layer=False):
        fy, fz = next(it) if it is not None else (None, None)
        y = force(q(F.conv2d(a, q(P[conv + ".weight"]), None, stride, k // 2)), fy)
        if ibn_layer:
            half = y.shape[1] // 2
            z = torch.cat((F.instance_norm(y[:, :half], None, None, P[name + ".IN.weight"], P[name + ".IN.bias"], True, 0.1, eps),
                           batch_norm(y[:, half:], name + ".BN")), 1)
        else:
            z = batch_norm(y, name)
        if res is not None:
            z = z + res
        return force(q(F.relu(z) if relu else z), fz)

    a = conv_bn(q(x.double()), "conv1", "bn1", 7, 2, relu=ibn)  # resnet.py:125: no ReLU after the stem; IBN-a has one
    a = F.max_pool2d(a, 3, 2, 1)
    for li, (planes, nblk) in enumerate(zip((64, 128, 256, 512), layers), start=1):
        stride0 = 1 if li == 1 else (last_stride if li == 4 else 2)
        for bi in range(nblk):
            p = f"layer{li}.{bi}"
            stride = stride0 if bi == 0 else 1
            o1 = conv_bn(a, p + ".conv1", p + ".bn1", 1, 1, ibn_layer=ibn and planes != 512)
            o2 = conv_bn(o1, p + ".conv2", p + ".bn2", 3, stride)
            res = a
            if bi == 0:
                res = conv_bn(a, p + ".downsample.0", p + ".downsample.1", 1, stride, relu=False)
            a = conv_bn(o2, p + ".conv3", p + ".bn3", 1, 1, res=res)
    feat = a.mean(dim=(2, 3))
    grads = None
    if dfeat is not None:
        (feat * dfeat.double()).sum().backward()
        grads = {k: v.grad for k, v in P.items()}
    return feat.detach(), grads, running


def augment_batch(images_u8, params, pixel_mean=(0.485, 0.456, 0.406), pixel_std=(0.229, 0.224, 0.225), pad=10):
    """datasets/transforms/build.py:18-27 after T.Resize, per image with GIVEN random draws (params int [B, 8] =
    flip, crop_top, crop_left, erase_row, erase_col, erase_h, erase_w, is_real): hflip -> Pad(pad, fill 0) ->
    crop to the original size -> ToTensor (/255) -> Normalize -> RandomErasing (random_erasing.py:44-51: the erased
    rectangle takes the RAW pixel mean, written after normalisation).  Mock images (is_real = 0) are all zeros
    (datasets/bases.py:378-391).  images_u8: uint8 [B, H, W, 3] -> float32 [B, 3, H, W]."""
    imgs = torch.as_tensor(images_u8)
    B, H, W, _ = imgs.shape
    mean = torch.tensor(pixel_mean, dtype=torch.float32)[:, None, None]
    std = torch.tensor(pixel_std, dtype=torch.float32)[:, None, None]
    out = torch.zeros(B, 3, H, W)
    for b in range(B):
        flip, top, left, er, ec, eh, ew, real = [int(v) for v in params[b]]
        if not real:
            continue
        im = imgs[b].permute(2, 0, 1)
        if flip:
            im = im.flip(2)
        im = F.pad(im, (pad, pad, pad, pad), value=0)[:, top:top + H, left:left + W]
        t = (im.float() / 255.0 - mean) / std
        if eh > 0:
            for c in range(3):
                t[c, er:er + eh, ec:ec + ew] = pixel_mean[c]
        out[b] = t
    return out


# --------------------------------------------------------------------------------------
# synthetic workloads shared by tests / bench (SURVEY 8d "Synthetic inputs")
# --------------------------------------------------------------------------------------


def synth_retrieval(num_q, num_g, num_ids, dim=2048, sigma=3.0, seed=0, num_cams=6, dyadic=False):
    """Clustered unit vectors: id centres c ~ N(0,I); sample = normalize(c_pid + sigma*N(0,I)).
    dyadic=True instead draws features on a coarse dyadic grid ({-1,-.5,0,.5,1}/8) so every
    dot product and norm is exact in fp32 AND in the fp16-split tensor-core arithmetic
    (bit-exact rank fixtures, SURVEY section 7 'hard parts')."""
    g = torch.Generator().manual_seed(seed)
    n = num_q + num_g
    pids = torch.randint(0, num_ids, (n,), generator=g)
    cams = torch.randint(0, num_cams, (n,), generator=g)
    if dyadic:
        centres = torch.randint(-2, 3, (num_ids, dim), generator=g).float()
        noise = torch.randint(-2, 3, (n, dim), generator=g).float()
        keep = (torch.rand(n, dim, generator=g) < 0.5).float()
        feats = (centres[pids] * keep + noise * (1 - keep)) / 16.0
    else:
        centres = torch.randn(num_ids, dim, generator=g)
        feats = centres[pids] + sigma * torch.randn(n, dim, generator=g)
        feats = F.normalize(feats, dim=1)
    return feats, pids.numpy().astype(np.int64), cams.numpy().astype(np.int64)


def synth_batch(P, K, dim=2048, num_classes=751, seed=0, pad_fraction=0.0, scale=1.0, pid_offset=0.15):
    """A CTL step's post-trunk inputs honouring the batch contract A0: pid-major blocks of K,
    padded (isReal=False, zero image -> here: features of a zero image are whatever the
    trunk gives; synthetic F rows are kept random) rows at the END of a pid's block, every
    pid keeps >= 2 real rows (datasets/bases.py:360)."""
    g = torch.Generator().manual_seed(seed)
    B = P * K
    pid_pool = torch.randperm(num_classes, generator=g)[:P]
    labels = pid_pool.repeat_interleave(K)
    feats = scale * torch.randn(B, dim, generator=g)
    feats = feats + scale * pid_offset * torch.randn(P, dim, generator=g).repeat_interleave(K, 0)
    is_real = torch.ones(B, dtype=torch.bool)
    if pad_fraction > 0:
        npad = max(1, int(round(P * pad_fraction)))
        for c in torch.randperm(P, generator=g)[:npad].tolist():
            drop = int(torch.randint(1, max(2, min(3, K - 1)), (1,), generator=g))
            drop = min(drop, K - 2)
            if drop > 0:
                is_real[c * K + K - drop : (c + 1) * K] = False
    return feats, labels, is_real
