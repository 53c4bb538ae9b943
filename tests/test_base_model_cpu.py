"""CPU: the base-model oracle (oracle/base_oracle.py) against the golden vectors the UNMODIFIED reference's
train_base_model.CTLModel.training_step produced, and the host side of the base-model loss ABI."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden
from oracle import ctl_oracle as O
from oracle.base_oracle import BASE_CASES, base_step_losses
from oracle.make_golden import DIM, NUM_CLASSES, checksum, head_state


def _close(a, b, rtol, atol=0.0):
    np.testing.assert_allclose(np.asarray(a), np.asarray(b), rtol=rtol, atol=atol)


def variant_kwargs(solver_over):
    """SOLVER overrides of a golden case -> base_step_losses keywords."""
    kw = {}
    if "DISTANCE_FUNC" in solver_over:
        kw["dist_func"] = solver_over["DISTANCE_FUNC"]
    if "MARGIN" in solver_over:
        kw["margin"] = solver_over["MARGIN"]
    return kw


@pytest.mark.parametrize("name", list(BASE_CASES))
def test_base_step_losses_match_reference(name):
    """Same tolerances as tests/test_oracle_golden.py::test_ctl_step_losses_match_reference."""
    g = load_golden(f"base_loss_{name}.npz")
    (P, K, pad, seed, scale), over = BASE_CASES[name]
    feats, labels, is_real = O.synth_batch(P, K, DIM, NUM_CLASSES, seed, pad, scale)
    _close(checksum(feats), g["in_checksum"], 1e-12)
    assert np.array_equal(is_real.numpy(), g["is_real"]) and np.array_equal(labels.numpy(), g["labels"])
    hs = head_state(seed)
    feats = feats.clone().requires_grad_(True)
    centers = hs["centers"].clone().requires_grad_(True)
    bn_w = hs["bn_weight"].clone().requires_grad_(True)
    fc_w = hs["fc_weight"].clone().requires_grad_(True)
    run_mean, run_var = torch.zeros(DIM), torch.ones(DIM)
    out = base_step_losses(feats, labels, is_real, centers, bn_w, hs["bn_bias"], fc_w, running_mean=run_mean,
                           running_var=run_var, **variant_kwargs(over))
    for key in ("total", "xent", "triplet", "center", "dist_ap", "dist_an"):
        _close(float(out[key].detach()), float(g[key]), 2e-5)
    out["total"].backward()
    # the feature gradient is stored as a row sample (mock rows included) plus checksums of the whole tensor
    gscale = float(g["grad_feats_abs_max"])
    _close(feats.grad[torch.from_numpy(g["grad_feats_rows_idx"])].numpy(), g["grad_feats_rows"], 1e-4, 1e-5 * gscale)
    _close(float(feats.grad.abs().max()), gscale, 1e-4)
    cs = checksum(feats.grad)
    assert abs(cs[0] - g["grad_feats_checksum"][0]) < 1e-5 * gscale * feats.numel() ** 0.5  # signed sum: absolute
    _close(cs[1], g["grad_feats_checksum"][1], 1e-4)
    rows = torch.from_numpy(g["grad_centers_rows_idx"])
    # the reference rescales centers.grad by 1/CENTER_LOSS_WEIGHT (train_base_model.py:80-81)
    gc = centers.grad[rows].numpy() / 5e-4
    _close(gc, g["grad_centers_rows"], 1e-4, 1e-6 * np.abs(g["grad_centers_rows"]).max())
    _close(float(centers.grad.abs().sum()) / 5e-4, float(g["grad_centers_abs_sum"]), 1e-4)
    _close(bn_w.grad.numpy(), g["grad_bn_weight"], 1e-3, 1e-5 * np.abs(g["grad_bn_weight"]).max())
    _close(fc_w.grad[rows].numpy(), g["grad_fc_rows"], 1e-3, 1e-5 * np.abs(g["grad_fc_rows"]).max())
    _close(run_mean.numpy(), g["bn_running_mean"], 1e-4, 1e-6)
    _close(run_var.numpy(), g["bn_running_var"], 1e-4, 1e-6)


def test_base_step_differs_from_ctl_step_on_padded_batches():
    """The two steps share trunk and head but not their row sets: on a batch with mock rows the base step's center loss
    and head see every row (train_base_model.py:67-73), the CTL step's only the real ones."""
    ctl = load_golden("loss_p8k4_pad.npz")
    base = load_golden("base_loss_p8k4_pad.npz")
    assert not bool(base["is_real"].all())
    assert float(base["center"]) != pytest.approx(float(ctl["center"]), rel=1e-3)
    assert float(base["xent"]) != pytest.approx(float(ctl["xent"]), rel=1e-3)
    real = load_golden("base_loss_p8k4_real.npz")
    real_ctl = load_golden("loss_p8k4_real.npz")
    for key in ("xent", "triplet", "center"):  # without mock rows the shared parts agree
        _close(float(real[key]), float(real_ctl[key]), 1e-6)


def test_base_loss_config_matches_header():
    """BaseLossConfig's ctypes fields are struct ctl_base_loss_config's, in order and type."""
    from ctl_b200 import _native as N

    header = open(os.path.join(ROOT, "include", "ctl_b200.h")).read()
    body = re.search(r"typedef struct ctl_base_loss_config \{(.*?)\} ctl_base_loss_config;", header, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            ctype, names = decl.split(None, 1)
            fields += [(n.strip(), ctype) for n in names.split(",")]
    ctypes_of = {"int32_t": ctypes.c_int32, "float": ctypes.c_float}
    assert [(n, ctypes_of[t]) for n, t in fields] == list(N.BaseLossConfig._fields_)


def test_base_loss_workspace_bytes_needs_no_device():
    """Workspace sizing is host arithmetic: positive for a valid shape, 0 (invalid argument) below two rows; the cosine
    variant needs the normalised rows on top."""
    from ctl_b200 import _native as N

    L = N.lib()

    def ws(B, cosine=0):
        cfg = N.BaseLossConfig(B, 2048, 751, 0.5, 0, cosine, 5e-4, 1.0, 1.0, 1e-5, 0.1, 0.1)
        return L.ctl_base_loss_workspace_bytes(ctypes.byref(cfg))

    assert ws(256) > 4 * (256 * 751 + 4 * 256 * 2048)
    assert ws(256, cosine=1) >= ws(256) + 4 * 256 * 2048
    assert ws(1) == 0 and b"bad dims" in L.ctl_last_error()
