"""ctypes binding of libctl_b200.so (the C ABI declared in include/ctl_b200.h).

The library is built in-tree by ``csrc/build.sh`` (``__graft_entry__.build()``); it is NOT
optional: there is no CPU or PyTorch fallback behind any compute entry point, and a missing
library or a non-sm_90 device raises here.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libctl_b200.so")

CTL_DIST_EUCLIDEAN = 0
CTL_DIST_COSINE = 1
CTL_FLAG_NORMALIZE = 2
CTL_DIST_SQRT = 4
CTL_BLOCK_BOTTLENECK = 0
CTL_BLOCK_BASIC = 1

_ERRORS = {
    -1: ValueError,   # CTL_ERR_INVALID_ARGUMENT
    -2: RuntimeError,  # CTL_ERR_WORKSPACE
    -3: NotImplementedError,  # CTL_ERR_UNSUPPORTED
    -4: OverflowError,  # CTL_ERR_CAPACITY
    -5: RuntimeError,  # CTL_ERR_NO_DEVICE
}

_p = C.c_void_p
_i64 = C.c_int64
_i32 = C.c_int32
_sz = C.c_size_t

_f = C.c_float


class LossConfig(C.Structure):
    """struct ctl_loss_config (include/ctl_b200.h)."""

    _fields_ = [("B", _i32), ("D", _i32), ("P", _i32), ("K", _i32), ("C", _i32), ("margin", _f),
                ("center_weight", _f), ("xent_weight", _f), ("triplet_weight", _f), ("ctl_weight", _f),
                ("bn_eps", _f), ("bn_momentum", _f), ("label_smooth", _f)]


_cfgp = C.POINTER(LossConfig)


class BaseLossConfig(C.Structure):
    """struct ctl_base_loss_config (include/ctl_b200.h)."""

    _fields_ = [("B", _i32), ("D", _i32), ("C", _i32), ("margin", _f), ("soft_margin", _i32), ("cosine", _i32),
                ("center_weight", _f), ("xent_weight", _f), ("triplet_weight", _f), ("bn_eps", _f),
                ("bn_momentum", _f), ("label_smooth", _f)]


_bcfgp = C.POINTER(BaseLossConfig)


class PassDesc(C.Structure):
    """struct ctl_pass_desc (include/ctl_b200.h)."""

    _fields_ = [("dist_out", _p), ("ld_out", _i64), ("gmin", _p), ("tau", _p), ("cand_keys", _p),
                ("cand_count", _p), ("cand_cap", _i32), ("q_pid", _p), ("q_cam", _p), ("g_pid", _p),
                ("g_cammask", _p), ("pos_keys", _p), ("pos_count", _p), ("max_pos", _i32), ("thr_keys", _p),
                ("thr_count", _p), ("buckets", _p), ("overflow", _p), ("g_index_offset", _i64),
                ("tile_list", _p), ("g_index_map", _p)]

class NamedTensor(C.Structure):
    """struct ctl_named_tensor (include/ctl_b200.h)."""

    _fields_ = [("name", C.c_char_p), ("data", _p), ("numel", _i64)]


class JpegDesc(C.Structure):
    """struct ctl_jpeg_desc (include/ctl_b200.h)."""

    _fields_ = [("h", _i32), ("w", _i32), ("scan_begin", C.c_uint32), ("scan_end", C.c_uint32),
                ("dqt", C.c_uint32 * 3), ("dht_dc", C.c_uint32 * 3), ("dht_ac", C.c_uint32 * 3),
                ("restart_interval", C.c_uint16), ("ncomp", C.c_uint8), ("dqt16", C.c_uint8),
                ("hs", C.c_uint8 * 3), ("vs", C.c_uint8 * 3), ("reserved", C.c_uint8 * 2)]


class JpegEntry(C.Structure):
    """struct ctl_jpeg_entry (include/ctl_b200.h)."""

    _fields_ = [("offset", _i64), ("nbytes", _i64), ("kind", _i32), ("reserved", _i32), ("desc", JpegDesc)]


CTL_JPEG_ENTRY_JPEG = 0
CTL_JPEG_ENTRY_RAW = 1
CTL_JPEG_ENTRY_MOCK = 2


# name -> (restype, argtypes); kept in one table so tests can check it against the header
SIGNATURES = {
    "ctl_last_error": (C.c_char_p, []),
    "ctl_abi_version": (C.c_int, []),
    "ctl_device_check": (C.c_int, []),
    "ctl_planes_bytes": (_sz, [_i64, _i32]),
    "ctl_planes_build": (C.c_int, [_p, _i64, _i32, _i32, _p, _p]),
    "ctl_dist_matrix": (C.c_int, [_p, _i64, _p, _i64, _i32, _i32, _p, _i64, _p]),
    "ctl_sort_key_rows": (C.c_int, [_p, _p, _i64, _i32, _p]),
    "ctl_eval_finalize_packed": (C.c_int, [_p, _p, _i64, _i32, _p, _p, _p, _p, _p]),
    "ctl_dist_pass": (C.c_int, [_p, _i64, _p, _i64, _i32, _i32, C.POINTER(PassDesc), _p]),
    "ctl_topk_plan": (C.c_int, [_i64, _i32, C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i32), C.POINTER(_i32)]),
    "ctl_select_tau": (C.c_int, [_p, _i64, _i32, _i32, _i32, _p, _p]),
    "ctl_dist_worklist_bytes": (_sz, [_i64, _i64]),
    "ctl_dist_subset_stride": (C.c_int, [_i64, _i32]),
    "ctl_dist_worklist": (C.c_int, [_p, _i64, _p, _i64, _i32, _p, _p]),
    "ctl_fill_f32": (C.c_int, [_p, _i64, C.c_float, _p]),
    "ctl_topk_emit": (C.c_int, [_p, _p, _i64, _i32, _i32, _p, _p, _p, _p]),
    "ctl_key_encode": (C.c_uint64, [C.c_float, C.c_uint32]),
    "ctl_key_decode": (None, [C.c_uint64, C.POINTER(C.c_float), C.POINTER(C.c_uint32)]),
    "ctl_eval_matrix_collect": (C.c_int, [_p, _i64, _i64, _i64, _p, _p, _p, _p, _i32, _p, _p, _p, _p]),
    "ctl_eval_matrix_count": (C.c_int, [_p, _i64, _i64, _i64, _p, _p, _p, _p, _i32, _p, _p, _p, _p]),
    "ctl_rerank_plan": (C.c_int, [_i64, _i64, _i32, _i32] + [C.POINTER(_i32)] * 4),
    "ctl_rerank_workspace_bytes": (_sz, [_i64, _i64, _i32, _i32]),
    "ctl_rerank": (C.c_int, [_p, _i64, _i64, _i32, _i32, _i32, _i32, _f, _p, _i64, _p, _p, _sz, _p]),
    "ctl_rerank_rank": (C.c_int, [_p, _i64, _i64, _i32, _p, _p, _p]),
    "ctl_rerank_expand": (C.c_int, [_p, _i64, _i64, _p, _i32, _i32, _p, _p, _p, _p]),
    "ctl_rerank_qe": (C.c_int, [_p, _i64, _i32, _i32, _p, _p, _p, _p, _p, _p, _p]),
    "ctl_rerank_invert": (C.c_int, [_i64, _i64, _p, _p, _p, _i32, _p, _p, _p, _p, _p]),
    "ctl_rerank_jaccard": (C.c_int, [_i64, _i64, _p, _p, _p, _i32, _p, _p, _p, _p, _i64, _f, _p, _i64, _p]),
    "ctl_rerank_topk_workspace_bytes": (_sz, [_i64, _i64, _i32, _i32, _i32, _i32, _i64]),
    "ctl_rerank_topk": (C.c_int, [_p, _i64, _i64, _i32, _i32, _i32, _i32, _f, _i32, _i64, _p, _p,
                                  _p, _p, _p, _p, _i32, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "ctl_rerank_dist_rows": (C.c_int, [_p, _i64, _i32, _i32, _i64, _i64, _i64, _i64, _p, _p, _i64, _p]),
    "ctl_rerank_rank_rows": (C.c_int, [_p, _i64, _i64, _i64, _i64, _i32, _p, _p, _p, _p]),
    "ctl_rerank_expand_rows": (C.c_int, [_p, _i64, _i64, _i64, _i64, _p, _i32, _i32, _p, _p, _p, _p]),
    "ctl_rerank_jaccard_rows": (C.c_int, [_i64, _i64, _i64, _i64, _p, _p, _p, _i32, _p, _p, _p, _p, _i64, _f, _p,
                                          _i64, _p]),
    "ctl_rerank_topk_rows": (C.c_int, [_p, _i64, _i64, _i64, _i64, _i32, _p, _p, _p]),
    "ctl_segment_mean": (C.c_int, [_p, _i64, _i32, _p, _p, _i64, _p, _p]),
    "ctl_loss_workspace_bytes": (_sz, [_cfgp]),
    "ctl_loss_step": (C.c_int, [_cfgp] + [_p] * 14 + [_p, _sz, _p]),
    "ctl_triplet_workspace_bytes": (_sz, [_i32, _i32]),
    "ctl_triplet_step": (C.c_int, [_p, _i32, _i32, _p, _p, _f, _p, _p, _p, _p, _p, _sz, _p]),
    "ctl_triplet_step_ex": (C.c_int, [_p, _i32, _i32, _p, _p, _f, _i32, _i32, _p, _p, _p, _p, _p, _sz, _p]),
    "ctl_center_loss_step": (C.c_int, [_p, _i32, _i32, _p, _p, _i32, _p, _p, _p, _p, _sz, _p]),
    "ctl_xent_smooth_step": (C.c_int, [_p, _i32, _i32, _p, _f, _p, _p, _p, _sz, _p]),
    "ctl_base_loss_workspace_bytes": (_sz, [_bcfgp]),
    "ctl_base_loss_step": (C.c_int, [_bcfgp] + [_p] * 14 + [_p, _sz, _p]),
    "ctl_conv2d_nhwc_f16": (C.c_int, [_p, _i32, _i32, _i32, _i32, _p, _p, _p, _p, _i32, _i32, _i32, _i32, _i32, _p]),
    "ctl_conv1x1_dual_nhwc_f16": (C.c_int, [_p, _i32, _p, _i32, _i32, _i32, _i32, _i32, _p, _p, _p, _i32, _i32, _p]),
    "ctl_conv3x3_dual_nhwc_f16": (C.c_int, [_p, _i32, _p, _i32, _i32, _i32, _i32, _i32, _p, _p, _p, _i32, _i32, _p]),
    "ctl_conv1x1_chain_supported": (_i32, [_i32, _i32]),
    "ctl_conv1x1_chain_nhwc_f16": (C.c_int, [_p, _i32, _p, _i32, _i32, _i32, _i32, _i32, _p, _p, _p, _p, _i32, _p, _p,
                                             _i32, _i32, _p, _p]),
    "ctl_trunk_create": (C.c_int, [C.POINTER(_p), _i32, _i32, _i32, C.POINTER(_i32)]),
    "ctl_trunk_feature_dim": (_i32, [_p]),
    "ctl_trunk_destroy": (None, [_p]),
    "ctl_weights_pack": (C.c_int, [_p, C.POINTER(NamedTensor), _i32, _p]),
    "ctl_embed_workspace_bytes": (_sz, [_p, _i32, _i32, _i32]),
    "ctl_embed_forward": (C.c_int, [_p, _p, _i32, _i32, _i32, _p, _p, _p, _sz, _p]),
    "ctl_embed_stem": (C.c_int, [_p, _p, _i32, _i32, _i32, C.POINTER(_f), C.POINTER(_f), _p, _p, _sz, _p]),
    "ctl_embed_blocks": (C.c_int, [_p, _p, _i32, _i32, _i32, _p, _p, _sz, _p]),
    "ctl_embed_head": (C.c_int, [_p, _p, _i32, _i32, _p, _p, _p]),
    "ctl_embed_launches": (_i32, [_p]),
    "ctl_trainer_create": (C.c_int, [C.POINTER(_p), _i32, _i32, _i32, C.c_float, C.POINTER(_i32)]),
    "ctl_trainer_feature_dim": (_i32, [_p]),
    "ctl_trainer_destroy": (None, [_p]),
    "ctl_trainer_bind": (C.c_int, [_p, C.POINTER(NamedTensor), _i32, C.POINTER(NamedTensor), _i32]),
    "ctl_train_workspace_bytes": (_sz, [_p, _i32, _i32, _i32]),
    "ctl_train_forward": (C.c_int, [_p, _p, _i32, _i32, _i32, _p, _p, _sz, _p]),
    "ctl_train_backward": (C.c_int, [_p, _p, C.c_float, _p, _sz, _p]),
    "ctl_train_saved": (C.c_int, [_p, _i32, C.POINTER(_p), C.POINTER(_p), C.POINTER(_i32)]),
    "ctl_stem_conv7x7_tc": (C.c_int, [_p, _i32, _i32, _i32, _p, _p, _i32, _p, _p]),
    "ctl_stem_pad_bytes": (C.c_size_t, [_i32, _i32, _i32]),
    "ctl_stem_pool_fused": (C.c_int, [_p, _i32, _i32, _i32, _p, _p, _p, _i32, _p, _p]),
    "ctl_stem_pool_fused_u8": (C.c_int, [_p, _i32, _i32, _i32, C.POINTER(C.c_float), C.POINTER(C.c_float), _p, _p, _p, _i32, _p, _p]),
    "ctl_maxpool3x3s2_nhwc_f16": (C.c_int, [_p, _i32, _i32, _i32, _i32, _p, _p]),
    "ctl_gap_bn_nhwc_f16": (C.c_int, [_p, _i32, _i32, _i32, _p, _p, _p, _p, _p]),
    "ctl_instnorm_relu_nhwc_f16": (C.c_int, [_p, _i32, _i32, _i32, _i32, _p, _p, _f, _p]),
    "ctl_bn_workspace_bytes": (C.c_size_t, [C.c_int64, _i32]),
    "ctl_bn_train_forward_nhwc_f16": (C.c_int, [_p, C.c_int64, _i32, _i32, _p, _p, _f, _f, _p, _p, _p, _i32, _p, C.c_size_t, _p, _p, _p, _p]),
    "ctl_bn_train_backward_nhwc_f16": (C.c_int, [_p, _p, _p, C.c_int64, _i32, _i32, _p, _p, _p, _f, _p, C.c_size_t, _p, _p, _p, _p, _p]),
    "ctl_instnorm_train_forward_nhwc_f16": (C.c_int, [_p, _i32, _i32, _i32, _i32, _p, _p, _f, _p, _p, _p, _p]),
    "ctl_instnorm_train_backward_nhwc_f16": (C.c_int, [_p, _p, _p, _i32, _i32, _i32, _i32, _p, _p, _p, _f, _p, _p, _p, _p]),
    "ctl_gap_backward_nhwc_f16": (C.c_int, [_p, _i32, _i32, _i32, _f, _p, _p]),
    "ctl_maxpool3x3s2_backward_nhwc_f16": (C.c_int, [_p, _p, _i32, _i32, _i32, _i32, _p, _p]),
    "ctl_maxpool3x3s2_argmax_nhwc_f16": (C.c_int, [_p, _i32, _i32, _i32, _i32, _p, _p, _p]),
    "ctl_maxpool3x3s2_backward_argmax_nhwc_f16": (C.c_int, [_p, _p, _i32, _i32, _i32, _i32, _p, _p]),
    "ctl_upsample2_zero_nhwc_f16": (C.c_int, [_p, _i32, _i32, _i32, _i32, _p, _p, _p]),
    "ctl_stem_im2col_f16": (C.c_int, [_p, _i32, _i32, _i32, _p, _p]),
    "ctl_augment_batch_u8": (C.c_int, [_p, _i32, _i32, _i32, _i32, _p, _p, _p, _p, _p]),
    "ctl_resize_bilinear_u8_workspace_bytes": (_sz, [_i64, _i32, _i32]),
    "ctl_resize_bilinear_u8": (C.c_int, [_p, _i64, _p, _i64, _i32, _i32, _p, _p, _p, _sz, _p]),
    "ctl_jpeg_parse": (C.c_int, [_p, _i64, C.POINTER(JpegDesc), C.POINTER(_i32), C.POINTER(_i32)]),
    "ctl_jpeg_decode_workspace_bytes": (_sz, [_p, _i64]),
    "ctl_jpeg_decode": (C.c_int, [_p, _i64, _p, _i64, _p, _p, _i64, _p, _p, _sz, _p]),
    "ctl_resize_linear_cv_u8": (C.c_int, [_p, _i64, _p, _i64, _i32, _i32, _p, _p, _p]),
    "ctl_visrank_compose": (C.c_int, [_p, _i64, _i32, _i32, _p, _i64, _i64, _i32, _p, _p, _p]),
    "ctl_visrank_select": (C.c_int, [_p, _i64, _i32, _p, _p, _p, _p, _i64, _i32, _p, _p, _p, _p]),
    "ctl_adam_multi_step": (C.c_int, [_p, _i32, C.c_int64, _f, _f, _f, _f, _f, C.c_int64, _f, _p, _p]),
    "ctl_sgd_step": (C.c_int, [_p, _p, C.c_int64, _f, _f, _p, _p]),
    "ctl_loss_scale_update": (C.c_int, [_p, _p, _p, _p, _f, _f, _f, _i32, _p]),
    "ctl_grad_check_multi": (C.c_int, [_p, _i32, C.c_int64, _f, _p, _p, _p]),
    "ctl_conv2d_wgrad_workspace_bytes": (C.c_size_t, [_i32, _i32, _i32, _i32, _i32, _i32, _i32]),
    "ctl_conv2d_wgrad_nhwc_f16": (C.c_int, [_p, _i32, _i32, _i32, _i32, _p, _i32, _i32, _i32, _p, C.c_size_t, _p, _p]),
    "ctl_conv2d_wgrad_nhwc_f16_ex": (C.c_int, [_p, _i32, _i32, _i32, _i32, _p, _i32, _i32, _i32, _p, C.c_size_t, _p, _f, _i32, _p]),
    "ctl_train_pack_weights": (C.c_int, [_p, _i32, C.c_int64, _p]),
}

_lib = None


def lib():
    """Loads the shared library once; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(centroids-reid_b200 has no CPU / PyTorch fallback)"
            )
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name, None)
            if fn is None:
                continue  # symbol checks live in tests/test_host_logic.py
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(rc: int):
    if rc == 0:
        return
    msg = lib().ctl_last_error().decode("utf-8", "replace")
    if rc < 0:
        raise _ERRORS.get(rc, RuntimeError)(f"ctl_b200 error {rc}: {msg}")
    raise RuntimeError(f"ctl_b200 CUDA error {rc}: {msg}")


def require_cuda(*tensors: torch.Tensor):
    """North-star contract: non-CUDA tensors raise, nothing silently runs on the host."""
    for t in tensors:
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise RuntimeError(
                "centroids-reid_b200 computes on a H100 only: expected CUDA tensors "
                f"(got {type(t).__name__}{'' if not isinstance(t, torch.Tensor) else ' on ' + str(t.device)})"
            )
    check(lib().ctl_device_check())


def ptr(t):
    return 0 if t is None else t.data_ptr()


def stream_ptr():
    return torch.cuda.current_stream().cuda_stream
