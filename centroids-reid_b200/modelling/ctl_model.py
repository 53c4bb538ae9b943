"""Drop-in for the tensor part of modelling/bases.py (ModelBase) and train_ctl_model.py
(CTLModel.training_step): same attribute names (backbone, bn, fc_query, center_loss,
contrastive_loss, xent), same hook signatures, the arithmetic on the H100 kernels.

pytorch_lightning is not a dependency of this package (and is absent from the build image): the class
derives from pl.LightningModule when PL is importable and from nn.Module otherwise.  Under PL the
hyper-parameters go through PL's own `hparams` setter + `save_hyperparameters` (modelling/bases.py:63-64),
and `training_step` performs the reference's complete manual-optimisation sequence
(train_ctl_model.py:38-179: warm-up LR, zero_grad, forward, losses, manual_backward, opt.step, center
gradient rescale, opt_center.step) whenever optimizers are attached -- by a Trainer (`self.optimizers()`)
or explicitly (`attach_optimizers`).  Without attached optimizers it returns the loss only and the caller
drives `backward()` / `optimizer_step_manual()` itself (bench.py, tests).  The PL path is exercised here
with a stub LightningModule (tests/test_host_logic.py); it has never run under a real pytorch_lightning.
"""
from __future__ import annotations

import os

import numpy as np
import torch
from torch import nn

from .. import _native as N
from .. import reduce as _reduce
from .. import retrieval as _R
from ..losses._fn import CTLStepFn, raise_if_poisoned
from ..losses.center_loss import CenterLoss
from ..losses.triplet_loss import CrossEntropyLabelSmooth, TripletLoss
from .baseline import Baseline, embed

try:  # pragma: no cover - PL is absent in the build image
    import pytorch_lightning as _pl

    _Base = _pl.LightningModule
except Exception:  # noqa: BLE001
    _Base = nn.Module

LOSS_NAMES = ("total", "query_xent", "query_triplet", "query_center", "centroid_triplet", "step_dist_ap",
              "step_dist_an", "l2_mean_centroid")


def ctl_losses_composed(module, features, class_labels, is_real):
    """train_ctl_model.py:54-152 for the TripletLoss variants the fused step does not cover (SOLVER.DISTANCE_FUNC =
    'cosine', SOLVER.MARGIN = None -> SoftMarginLoss): the same arithmetic assembled from the stand-alone drop-in losses
    (each a fused forward+backward kernel behind torch.autograd) with the masks / centroid means in closed form
    (SURVEY appendix A.1):  M_i[c, s] = (s != i) & R[c, i] & R[c, s],  centroid_i[c] = sum_s M_i[c, s] F[cK + s] / n_i[c],
    round i = TripletLoss over [queries F[cK + i] ; centroids_i], skipped unless more than one class has a centroid.
    Returns (total, parts[8]) like ctl_losses; this path synchronises (boolean row selection), the fused one does not."""
    hp = module.hparams
    K = int(hp.DATALOADER.NUM_INSTANCE)
    B, D = features.shape
    P = B // K
    S = hp.SOLVER
    real = is_real.bool()
    F3 = features.view(P, K, D)
    L2 = class_labels.view(P, K)
    R = real.view(P, K)
    lq, _, _ = module.contrastive_loss(features, class_labels, mask=real)
    lq = lq * S.QUERY_CONTRASTIVE_WEIGHT
    f_real, y_real = features[real], class_labels[real]
    center = S.CENTER_LOSS_WEIGHT * module.center_loss(f_real, y_real)
    xent = module.xent(module.fc_query(module.bn(f_real)), y_real) * S.QUERY_XENT_WEIGHT
    eye = torch.eye(K, dtype=torch.bool, device=features.device)
    M = (~eye)[:, None, :] & R.t()[:, :, None] & R[None, :, :]            # [round i, class c, slot s]
    n = M.sum(-1)                                                          # [K, P]
    cent = torch.einsum("ics,csd->icd", M.to(features.dtype), F3) / n.clamp(min=1)[..., None].to(features.dtype)
    valid_round = ((n > 0).sum(1) > 1).tolist()                            # train_ctl_model.py:113
    losses, aps, ans, l2s = [], [], [], []
    for i in range(K):
        if not valid_round[i]:
            continue
        q_sel = R[:, i]
        queries, labs = F3[:, i][q_sel], L2[:, i][q_sel]
        c_i = cent[i]
        c_i = c_i[c_i.abs().sum(1) > 1e-7]                                 # train_ctl_model.py:120-122
        loss_i, ap, an = module.contrastive_loss(torch.cat((queries, c_i)), torch.cat((labs, labs)))
        losses.append(loss_i)
        aps.append(ap.detach().mean())
        ans.append(an.detach().mean())
        l2s.append(c_i.detach().norm(dim=1).mean())
    ctl = torch.stack(losses).mean() * S.CENTROID_CONTRASTIVE_WEIGHT
    total = ctl + center + xent + lq
    parts = torch.stack([total.detach(), xent.detach(), lq.detach(), center.detach(), ctl.detach(),
                         torch.stack(aps).mean(), torch.stack(ans).mean(), torch.stack(l2s).mean()]).float()
    return total, parts


def ctl_losses(module, features, class_labels, is_real):
    """train_ctl_model.py:54-152 in one call: returns (total_loss tensor with autograd into
    features / centers / bn.weight / fc_query.weight, parts float32[8] on the device in
    LOSS_NAMES order).  No host synchronisation."""
    hp = module.hparams
    if hp.SOLVER.DISTANCE_FUNC != "euclidean" or hp.SOLVER.MARGIN is None:
        return ctl_losses_composed(module, features, class_labels, is_real)
    K = int(hp.DATALOADER.NUM_INSTANCE)
    B, D = features.shape
    if B % K != 0:
        raise ValueError(f"batch contract: B={B} must be P*K with K={K} (datasets/bases.py:346-406)")
    if not module.bn.training:
        raise NotImplementedError("the fused loss step normalises with BATCH statistics (nn.BatchNorm1d in train mode, as in "
                                  "the reference's training_step); call module.train() / module.bn.train() first")
    cfg = N.LossConfig(B, D, B // K, K, module.fc_query.weight.shape[0], float(hp.SOLVER.MARGIN),
                       float(hp.SOLVER.CENTER_LOSS_WEIGHT), float(hp.SOLVER.QUERY_XENT_WEIGHT),
                       float(hp.SOLVER.QUERY_CONTRASTIVE_WEIGHT), float(hp.SOLVER.CENTROID_CONTRASTIVE_WEIGHT),
                       float(module.bn.eps), float(module.bn.momentum), 0.1)
    total, parts = CTLStepFn.apply(features, module.center_loss.centers, module.bn.weight, module.fc_query.weight,
                                   module.bn.bias, module.bn.running_mean, module.bn.running_var, class_labels, is_real, cfg)
    # The kernels derive a row's class from its position (pid-major blocks of K, datasets/bases.py:346-406) and index the
    # centers by label: a violated contract comes back as a NaN with a payload.
    fused_step_done(module, parts, "CTL training step")
    return total, parts


def fused_step_done(module, parts, what):
    """Host bookkeeping after a fused loss step wrote the head's running statistics through raw pointers.  The step
    reports a violated batch contract as a NaN with a payload in parts[0]; the sampler's layout does not change between
    steps, so the (synchronising) check runs on the FIRST step of a module only; CTL_VALIDATE_BATCH=1 checks every step."""
    if module.bn.num_batches_tracked is not None:
        module.bn.num_batches_tracked += 1  # nn.BatchNorm1d.forward bookkeeping (the running statistics moved)
    from ..solver.build import _bump_version

    _bump_version([module.bn.running_mean, module.bn.running_var])  # written by the kernel through raw pointers
    if not module.__dict__.get("_ctl_batch_checked", False) or os.environ.get("CTL_VALIDATE_BATCH") == "1":
        raise_if_poisoned(parts[0], what)
        module.__dict__["_ctl_batch_checked"] = True


class CTLModel(_Base):
    """ModelBase.__init__ (modelling/bases.py:53-90) + CTLModel (train_ctl_model.py:27-36)."""

    def __init__(self, cfg=None, test_dataloader=None, **kwargs):
        super().__init__()
        hp = dict(cfg) if cfg is not None else {}
        hp.update(kwargs)
        if _Base is nn.Module:
            self.__dict__["hparams"] = _AttrDict(hp)
        else:
            # modelling/bases.py:63-64: PL 1.1.4's `hparams` is a property with a setter; assign through it and
            # register the values for checkpointing exactly like the reference
            try:
                from pytorch_lightning.utilities import AttributeDict as _PLAttrDict
            except Exception:  # noqa: BLE001
                _PLAttrDict = _AttrDict
            self.hparams = _PLAttrDict(hp)
            self.save_hyperparameters(self.hparams)
        if test_dataloader is not None:
            self.test_dataloader = test_dataloader
        self._ctl_optimizers = None
        self.backbone = Baseline(self.hparams)
        self.contrastive_loss = TripletLoss(self.hparams.SOLVER.MARGIN, self.hparams.SOLVER.DISTANCE_FUNC)
        d_model = self.hparams.MODEL.BACKBONE_EMB_SIZE
        if d_model != self.backbone.in_planes:
            # the loss kernels index bn / fc_query / centers by the feature width: a mismatch would be silently wrong
            raise ValueError(f"MODEL.BACKBONE_EMB_SIZE={d_model} but MODEL.NAME={self.hparams.MODEL.NAME!r} produces "
                             f"{self.backbone.in_planes}-wide features")
        self.xent = CrossEntropyLabelSmooth(num_classes=self.hparams.num_classes)
        self.center_loss = CenterLoss(num_classes=self.hparams.num_classes, feat_dim=d_model,
                                      use_gpu=torch.cuda.is_available())
        self.center_loss_weight = self.hparams.SOLVER.CENTER_LOSS_WEIGHT
        self.bn = torch.nn.BatchNorm1d(d_model)
        self.bn.bias.requires_grad_(False)  # bases.py:83-84
        self.fc_query = torch.nn.Linear(d_model, self.hparams.num_classes, bias=False)
        nn.init.normal_(self.fc_query.weight, std=0.001)  # weights_init_classifier, bases.py:29-34
        self.losses_names = ["query_xent", "query_triplet", "query_center", "centroid_triplet"]
        self.losses_dict = {n: [] for n in self.losses_names}

    # -- training ---------------------------------------------------------------------------
    def training_step_from_features(self, features, class_labels, is_real):
        """Everything of training_step after `_, features = self.backbone(x)`
        (train_ctl_model.py:59) up to and including the loss assembly (:150-152)."""
        total, parts = ctl_losses(self, features, class_labels, is_real)
        return {"loss": total, "parts": parts}

    def attach_optimizers(self, opt, opt_center):
        """Makes `training_step` a complete iteration outside a PL Trainer (the optimizers `configure_optimizers` built)."""
        self._ctl_optimizers = (opt, opt_center)

    def _step_optimizers(self):
        if self._ctl_optimizers is not None:
            return self._ctl_optimizers
        if _Base is not nn.Module and getattr(self, "trainer", None) is not None:
            return self.optimizers(use_pl_optimizer=True)  # train_ctl_model.py:39
        return None

    def training_step(self, batch, batch_idx, optimizer_idx=None):
        """train_ctl_model.py:38-179.  With optimizers attached (PL Trainer or `attach_optimizers`): the reference's whole
        manual-optimisation iteration, returning {"loss", "other": {step_dist_ap, step_dist_an, l2_mean_centroid}}.
        Without: forward + losses only, returning {"loss" (differentiable), "parts"}."""
        x, class_labels, camid, is_real = batch
        opts = self._step_optimizers()
        if opts is None:
            _, features = self.backbone(x)  # train mode: H100 training engine (differentiable w.r.t. the trunk parameters)
            return self.training_step_from_features(features, class_labels, is_real)
        opt, opt_center = opts
        epoch = int(getattr(getattr(self, "trainer", None), "current_epoch", 0) or 0)
        opt_center.zero_grad()
        opt.zero_grad()
        _, features = self.backbone(x)
        out = self.training_step_from_features(features, class_labels, is_real)
        total = out["loss"]
        if _Base is not nn.Module and getattr(self, "trainer", None) is not None:
            self.manual_backward(total, optimizer=opt)
        else:
            total.backward()
        self.optimizer_step_manual(opt, opt_center, epoch=epoch)
        return self._log_step(total, out["parts"].tolist())  # ONE read-back for everything the reference logs

    def _log_step(self, total, parts):
        """train_ctl_model.py:161-179: the parts the reference logs with float(...), from the host copy of `parts`."""
        for name, val in zip(self.losses_names, (parts[1], parts[2], parts[3], parts[4])):
            self.losses_dict[name].append(val)
        return {"loss": total.detach(), "other": {"step_dist_ap": parts[5], "step_dist_an": parts[6],
                                                  "l2_mean_centroid": parts[7]}}

    def configure_optimizers(self):
        """modelling/bases.py:97-100 with the fused optimizers of ctl_b200.solver.build."""
        from ..solver.build import build_optimizer, build_scheduler

        optimizers_list = build_optimizer(self.named_parameters(), self.hparams)
        self.lr_scheduler = build_scheduler(optimizers_list[0], self.hparams)
        return optimizers_list, self.lr_scheduler

    def optimizer_step_manual(self, opt, opt_center, epoch: int = 0):
        """The tail of train_ctl_model.py:154-159 after `manual_backward`: warm-up LR rule (bases.py:115-121),
        `opt.step()`, center gradients rescaled by 1 / CENTER_LOSS_WEIGHT, `opt_center.step()`; the packed eval
        weights are invalidated because the parameters changed."""
        from ..solver.build import apply_warmup_lr

        apply_warmup_lr(opt, epoch, self.hparams)
        scaler = self.backbone.loss_scaler
        if scaler is not None and scaler.enabled:
            # GradScaler.step / update without a host synchronisation: one pass over every gradient the optimizers are
            # about to consume (after any gradient all-reduce, so all ranks agree) raises a DEVICE flag; the optimizer
            # kernels skip themselves when it is set (Adam's moments are never poisoned); the scale backs off / grows on
            # the device; the step counters are corrected one step late (DynamicLossScaler.settle)
            scaler.settle(opt, opt_center)
            scaler.check([p.grad for p in self.parameters() if p.grad is not None])
            opt.skip_flag = opt_center.skip_flag = scaler.flag
        opt.step()
        for param in self.center_loss.parameters():
            param.grad.data *= 1.0 / self.hparams.SOLVER.CENTER_LOSS_WEIGHT
        opt_center.step()
        if scaler is not None and scaler.enabled:
            scaler.update()
        self.backbone.invalidate()

    # -- evaluation -------------------------------------------------------------------------
    def validation_step(self, batch, batch_idx):
        """modelling/bases.py:169-177."""
        self.backbone.eval()
        self.bn.eval()
        x, class_labels, camid, idx = batch
        with torch.no_grad():
            emb = embed(self, x)
        return {"emb": emb, "labels": class_labels, "camid": camid, "idx": idx}

    test_step = validation_step

    def validation_create_centroids(self, embeddings, labels, camids, respect_camids=False):
        """modelling/bases.py:179-262 (features stay on the device)."""
        return _reduce.validation_create_centroids(embeddings, labels, camids, self.hparams.num_query, respect_camids)

    @staticmethod
    def _calculate_centroids(vecs, dim=1):
        return _reduce._calculate_centroids(vecs, dim)

    def get_val_metrics(self, embeddings, labels, camids):
        """modelling/bases.py:264-297 without the loggers: returns (cmc, mAP, all_topk)."""
        hp = self.hparams
        respect = bool(hp.MODEL.KEEP_CAMID_CENTROIDS and hp.MODEL.USE_CENTROIDS)
        nq = hp.num_query
        emb = torch.as_tensor(embeddings).float()
        emb = emb if emb.is_cuda else emb.cuda(non_blocking=True)
        q_lab, g_lab = np.asarray(labels[:nq]), np.asarray(labels[nq:])
        go = _R.pid_order(g_lab) if len(g_lab) == emb.shape[0] - nq else None  # identity order: cheap collect pass
        qp = _R.build_planes(emb[:nq], hp.SOLVER.DISTANCE_FUNC, hp.TEST.FEAT_NORM, order=_R.pid_order(q_lab))
        gp = _R.build_planes(emb[nq:], hp.SOLVER.DISTANCE_FUNC, hp.TEST.FEAT_NORM, order=go)
        res = _R.evaluate_streamed(qp, gp, q_lab, g_lab, camids[:nq], camids[nq:], 50, respect)
        for top_k, kk in zip(res.all_topk, [1, 5, 10, 20, 50]):
            print("top-k, Rank-{:<3}:{:.1%}".format(kk, top_k))
        print(f"mAP: {res.mAP}")
        return res.cmc, res.mAP, res.all_topk

    def validation_epoch_end(self, outputs):
        """modelling/bases.py:299-318 (rank-0 gating and loggers are the Trainer's business)."""
        embeddings = torch.cat([x["emb"] for x in outputs]).detach()
        labels = torch.cat([x["labels"] for x in outputs]).detach().cpu().numpy()
        camids = torch.cat([x["camid"] for x in outputs]).detach().cpu().numpy()
        if self.hparams.MODEL.USE_CENTROIDS:
            print("Evaluation is done using centroids")
            embeddings, labels, camids = self.validation_create_centroids(
                embeddings, labels, camids, respect_camids=self.hparams.MODEL.KEEP_CAMID_CENTROIDS)
        return self.get_val_metrics(embeddings, labels, camids)

    test_epoch_end = validation_epoch_end


class _AttrDict(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v
