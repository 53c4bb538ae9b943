"""Drop-in for the reference's inference helpers (inference/inference_utils.py, create_embeddings.py,
get_similar.py): the data formats either side of the hot path.

Same names, arguments and on-disk formats:
  * `embeddings.npy`  float32 [N, 2048]   (create_embeddings.py:108)
  * `paths.npy`       str / object [N]    (create_embeddings.py:109; pids as numpy str_ when centroids are saved)
  * `results.npy`     pickled dict  query_path -> {"indices", "paths", "distances"}   (get_similar.py:121-137)
  * `query_embeddings.npy`, `query_paths.npy`

What changes underneath: `_inference` runs the H100 trunk engine (`modelling.baseline.embed`), `run_inference` keeps
the embeddings on the device and copies them to the host ONCE (the reference does one `.cpu().numpy()` per image,
inference_utils.py:123-125), `calculate_centroids` is the segmented-mean kernel, and `get_similar` streams
query x gallery distances into a per-query top-k without materialising the [Q, G] matrix or its argsort
(get_similar.py:112-119); with `topk == 0` the full matrix path of the reference is kept.
The image-folder datasets of the reference stay where they are.  A loader that ships file bytes as a JpegBatch
(datasets.transforms.pack_jpegs) has the JPEG decode and `T.Resize` run on the device, bit for bit Pillow's; one that
ships decoded images at native size as a RaggedImages has `T.Resize` run there.
"""
from __future__ import annotations

import logging
from pathlib import Path
from typing import Callable, Dict, List

import numpy as np
import torch

from .. import retrieval as R
from ..datasets.transforms import JpegBatch, RaggedImages, decode_batch, resize_batch
from ..modelling.baseline import embed
from ..reduce import calculate_centroids  # noqa: F401  (re-export: inference_utils.py:147-159)
from ..utils.reid_metric import get_dist_func

log = logging.getLogger(__name__)


def _inference(model, batch, use_cuda=True, normalize_with_bn=True, cfg=None):
    """inference_utils.py:104-113.  `model` exposes `.backbone` (ctl_b200 Baseline) and `.bn`.  `batch[0]` is the
    reference's float tensor [B, 3, H, W], or a RaggedImages of native-size images (datasets.transforms.pack_images):
    those are resized on the device to cfg.INPUT.SIZE_TEST (`T.Resize`, bit for bit PIL's) and embedded from uint8
    with cfg.INPUT.PIXEL_MEAN / PIXEL_STD (TrunkEngine.forward_u8), so the loader ships native-size bytes only.  A
    JpegBatch of file bytes (datasets.transforms.pack_jpegs) is first decoded on the device (decode_batch)."""
    if not use_cuda:
        raise RuntimeError("ctl_b200 has no CPU path (use_cuda=False); run the reference for CPU inference")
    data, _, filename = batch
    if isinstance(data, JpegBatch):
        if cfg is None:
            raise ValueError("_inference: a JpegBatch needs cfg (INPUT.SIZE_TEST, PIXEL_MEAN, PIXEL_STD)")
        data = decode_batch(data.to("cuda"))
    if isinstance(data, RaggedImages):
        if cfg is None:
            raise ValueError("_inference: a RaggedImages batch needs cfg (INPUT.SIZE_TEST, PIXEL_MEAN, PIXEL_STD)")
        with torch.no_grad():
            u8 = resize_batch(data.to("cuda"), cfg.INPUT.SIZE_TEST)
            eng = model.backbone.engine(bn_head=model.bn) if normalize_with_bn else model.backbone.engine()
            out = eng.forward_u8(u8, want_emb=normalize_with_bn, pixel_mean=tuple(cfg.INPUT.PIXEL_MEAN),
                                 pixel_std=tuple(cfg.INPUT.PIXEL_STD))
        return out["emb" if normalize_with_bn else "global_feat"], filename
    data = data.cuda(non_blocking=True)
    with torch.no_grad():
        if normalize_with_bn:
            feat = embed(model, data)
        else:
            feat = model.backbone.engine().forward(data)["global_feat"]
    return feat, filename


def run_inference(model, val_loader, cfg, print_freq, use_cuda=True):
    """inference_utils.py:116-131 -> (embeddings float32 [N, D] numpy, paths numpy array).  The loader yields float
    tensors as the reference's does, RaggedImages of native-size images (resized on the device, see _inference), or
    JpegBatch of file bytes (decoded and resized on the device)."""
    chunks, paths = [], []
    for pos, x in enumerate(val_loader):
        if pos % print_freq == 0:
            log.info(f"Number of processed images: {pos * cfg.TEST.IMS_PER_BATCH}")
        embedding, path = _inference(model, x, use_cuda, cfg=cfg)
        chunks.append(embedding)  # stays on the device; one D2H copy at the end
        paths.extend(list(path))
    if not chunks:
        return np.zeros((0, 0), dtype=np.float32), np.array(paths)
    dev = torch.cat(chunks, 0).float()
    host = torch.empty(dev.shape, dtype=torch.float32, pin_memory=True)
    host.copy_(dev, non_blocking=True)
    torch.cuda.current_stream().synchronize()
    return host.numpy().copy(), np.array(paths)


def create_pid_path_index(paths: List[str], func: Callable[[str], str]) -> Dict[str, list]:
    """inference_utils.py:134-144 (insertion-ordered pid -> row indices)."""
    index: Dict[str, list] = {}
    for idx, item in enumerate(paths):
        index.setdefault(func(item), []).append(idx)
    return index


def save_gallery(save_dir, embeddings, paths):
    """create_embeddings.py:103-109."""
    save_dir = Path(save_dir)
    save_dir.mkdir(exist_ok=True, parents=True)
    np.save(save_dir / "embeddings.npy", np.asarray(embeddings))
    np.save(save_dir / "paths.npy", np.asarray(paths))


def load_gallery(load_dir):
    """get_similar.py:93-97 -> (float32 tensor [G, D], paths array)."""
    load_dir = Path(load_dir)
    emb = torch.from_numpy(np.load(load_dir / "embeddings.npy", allow_pickle=True))
    return emb, np.load(load_dir / "paths.npy", allow_pickle=True)


def get_similar(embeddings, paths, embeddings_gallery, paths_gallery, dist_func_name="euclidean", topk=100,
                normalize_features=False, device="cuda"):
    """get_similar.py:99-130: optional L2-normalisation, distance, ascending ranks, top-k slice, and the result
    dict {query_path: {"indices", "paths", "distances"}}.  `topk == 0` returns every gallery id per query."""
    q = torch.as_tensor(np.asarray(embeddings) if not torch.is_tensor(embeddings) else embeddings).float().to(device)
    g = torch.as_tensor(np.asarray(embeddings_gallery) if not torch.is_tensor(embeddings_gallery)
                        else embeddings_gallery).float().to(device)
    paths_gallery = np.asarray(paths_gallery)
    n_g = g.shape[0]
    if topk and topk < n_g:
        idx, dst = R.topk_similar(q, g, int(topk), dist_func_name, bool(normalize_features))
        indices, distances = idx.cpu().numpy(), dst.cpu().numpy()
    else:
        # every id requested: the reference's full matrix + argsort (stable, so ties resolve by index like the
        # streamed path and the oracle)
        if normalize_features:
            q = torch.nn.functional.normalize(q, dim=1, p=2)
            g = torch.nn.functional.normalize(g, dim=1, p=2)
        distmat = get_dist_func(dist_func_name)(x=q, y=g).cpu().numpy()
        indices = np.argsort(distmat, axis=1, kind="stable")
        distances = np.take_along_axis(distmat, indices, axis=1)
    return {
        query_path: {"indices": indices[i, :], "paths": paths_gallery[indices[i, :]], "distances": distances[i, :]}
        for i, query_path in enumerate(paths)
    }


def save_results(save_dir, out, embeddings, paths):
    """get_similar.py:132-139."""
    save_dir = Path(save_dir)
    save_dir.mkdir(exist_ok=True, parents=True)
    np.save(save_dir / "results.npy", out)
    np.save(save_dir / "query_embeddings.npy", np.asarray(embeddings))
    np.save(save_dir / "query_paths.npy", np.asarray(paths))
