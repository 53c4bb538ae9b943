"""GPU: the fused stem (csrc/conv.cu: stem_pack_input_kernel / stem_pack_input_u8_kernel, then stem_pool_kernel) and the
eval handle's BatchNorm folding (csrc/trunk.cu: stem_pack_kernel, fold_pack_kernel with its IBN channel offset,
head_pack_kernel, and pack_dual's [W_last | Wd] bias sum), against float64 torch on the CPU.

  1. The fused stem's staging buffer [n][h+6][136][4] fp16, read back after the call, bit for bit: fp16(x) or
     fp16((u / 255 - mean) / std) in channels 0..2 of the interior, zero everywhere else (channel 3, the 3-pixel
     top / left border, the rows and columns past the image, the 256-byte slack), also after the fp32 and the uint8
     entry points have written the same buffer one after the other.
  2. conv 7x7 / 2 (+bias, optional ReLU) + maxpool 3x3 / 2 per element, on the fp16 operands the kernel reads, at every
     width class (w % 4 == 2 gives an odd conv width, whose last pool window is clamped on the right), at tile counts
     (n * h / 4 row pairs) around the SM count (CTAs that start inside an image and recompute the row pair above, at an
     image start, uneven ranges) and at the bench batches.
  3. The handle's stem (fused, from fp32 and uint8, and the tensor-core stem + max-pool) and head on BatchNorms with
     adversarial but bounded statistics: running_var 0 and 1e-7 (the folded scale is ~3 only because of eps),
     running_var 1e4, negative gamma, |running_mean| 30 with beta cancelling it to a bias of ~0.1.
  4. The same kind of statistics in every BatchNorm of ResNet18 and ResNet50-IBN-a, through the whole trunk.
  5. CPU self-checks (not marked gpu): the test's model of the staging layout and of the [28][64][8] weight operand
     is the convolution F.conv2d computes, and every plausible wrong fold moves the references of items 3 and 4 by at
     least 10x their tolerance, so that the GPU tests can fail.

Every output starts as NaN, so that an element a kernel never writes fails.  Budgets (u = 2^-24):
  - stem, per pooled element, max being 1-Lipschitz: 2^-10 maxpool(|conv + b|) + 2^-20 maxpool(conv(|x16|, |w16|)),
    the tensor-core stem budget of test_eval_kernels_gpu.py carried through the window max (the window max of |y|,
    not |max y|: without ReLU a window can be all negative).
  - stem against the float64 BatchNorm of the unfolded weights: that budget + 2^-11 maxpool(conv(|x16|, |w s|)) for
    the fp16 rounding of the folded weights + 2^-22 (|beta| + |mean s|) for the fp32 bias beta - mean s.
  - head: 2^-21 (|feat s| + |mean s| + |beta|), the fp32 roundings of s, of beta - mean s and of the fma.
  - trunk: 3e-3 of the feature scale against the fp16-rounding checkers, as test_trunk_gpu.py."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import basic_oracle as BO
from oracle import ctl_oracle as O

gpu = pytest.mark.gpu  # every GPU test carries it; the CPU self-checks of item 5 run under -m "not gpu"

EPS = 1e-5
WP = 136  # staging row pitch, pixels (S3_WP)
IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
# A mean / std per channel at which some u in [0, 255] gives (u / 255 - m) / s and (u / 255 - m) * (1 / s) different
# fp16 roundings (u = 122, 3 and 157); with ImageNet's the two agree after fp16 rounding for every u.
ODD_NORM = ((0.355, 0.497, 0.361), (0.225, 0.478, 0.395))
KEY_U8 = (0, 255, 122, 3, 157)  # written to every channel of the first pixels of image 0


def _n():
    from ctl_b200 import _native as N

    return N, N.lib()


def _bits(t):
    t = t.contiguous()
    return t.view({torch.float16: torch.int16, torch.float32: torch.int32}[t.dtype])


def _report(err, tol):
    bad = err > tol
    return (f"{int(bad.sum())} / {bad.numel()} off; max err/budget {float((err / tol).max()):.3f}; first bad index "
            f"{bad.nonzero()[0].tolist() if bad.any() else None}")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ===================================================================================================================
# host models: the staging layout, the weight operand, the float64 stem, the CTA ranges of stem_pool_kernel
# ===================================================================================================================
def _pool_shape(h, w):
    ho, wo = h // 2, w // 2  # even h, w: conv 7x7 / 2, pad 3
    return (ho - 1) // 2 + 1, (wo - 1) // 2 + 1


def _staged(x16):
    """fp16 [n, 3, h, w] -> the whole staging buffer ([n][h+6][136][4] and 128 fp16 of slack) as int16 bits."""
    n, _, h, w = x16.shape
    e = torch.zeros(n, h + 6, WP, 4, dtype=torch.float16)
    e[:, 3:h + 3, 3:w + 3, :3] = x16.permute(0, 2, 3, 1)
    return torch.cat((_bits(e).flatten(), torch.zeros(128, dtype=torch.int16)))


def _interior(buf, n, h, w):
    """staging buffer bits -> the fp16 input [n, 3, h, w] it holds."""
    e = buf[:n * (h + 6) * WP * 4].view(torch.float16).view(n, h + 6, WP, 4)
    return e[:, 3:h + 3, 3:w + 3, :3].permute(0, 3, 1, 2).contiguous()


def _where(i, n, h):
    """flat fp16 index into the staging buffer -> readable position."""
    if i >= n * (h + 6) * WP * 4:
        return f"slack element {i - n * (h + 6) * WP * 4}"
    i, ch = divmod(i, 4)
    i, px = divmod(i, WP)
    img, row = divmod(i, h + 6)
    return f"image {img}, padded row {row}, padded column {px}, channel {ch}"


def _normalize_u8(img, mean, std):
    """uint8 [n, h, w, 3] -> fp32 [n, 3, h, w] = (u / 255 - mean) / std, each operation one IEEE fp32 rounding
    (numpy divides; it never multiplies by a reciprocal)."""
    u = img.numpy().astype(np.float32) / np.float32(255)
    out = (u - np.asarray(mean, np.float32)) / np.asarray(std, np.float32)
    return torch.from_numpy(out).permute(0, 3, 1, 2).contiguous()


def _crops(n, h, w, seed):
    """random uint8 crops; image 0 starts with KEY_U8 in every channel and its bottom-right pixels are 0 and 255."""
    img = torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed))
    flat = img[0].view(h * w, 3)
    for i, v in enumerate(KEY_U8):
        flat[i] = v
    flat[-2], flat[-1] = 0, 255
    return img


def _unpack_w3(w3):
    """fused-stem operand [28][64][8] (chunk = r * 4 + s // 2, element = (s % 2) * 4 + ch) -> [64, 4, 7, 8] [o][ch][r][s]."""
    return w3.reshape(7, 4, 64, 2, 4).permute(2, 4, 0, 1, 3).reshape(64, 4, 7, 8)


def _conv_as_read(buf, w3, n, h, w):
    """The convolution stem_pool_kernel's wgmma windows compute, read straight off the staging buffer and the operand:
    conv output (oy, ox) = sum over r < 7, s < 8, ch < 4 of w[o][ch][r][s] * staged[2 oy + r][2 ox + s][ch]."""
    e = buf[:n * (h + 6) * WP * 4].view(torch.float16).view(n, h + 6, WP, 4).permute(0, 3, 1, 2).double()
    y = F.conv2d(e, _unpack_w3(w3).double(), None, 2)
    return y[:, :, :h // 2, :w // 2]


def _stem_ref(x16, w, b, relu, chunk=16):
    """float64 maxpool(act(conv(x16, w) + b)) and its budget (module docstring); x16, w exactly representable."""
    refs, tols = [], []
    for i in range(0, x16.shape[0], chunk):
        xd = x16[i:i + chunk].double()
        y = F.conv2d(xd, w.double(), b.double(), 2, 3)
        mag = F.max_pool2d(F.conv2d(xd.abs(), w.double().abs(), None, 2, 3), 3, 2, 1)
        refs.append(F.max_pool2d(y.clamp(min=0) if relu else y, 3, 2, 1))
        tols.append(2.0 ** -10 * F.max_pool2d(y.abs(), 3, 2, 1) + 2.0 ** -20 * mag)
    return torch.cat(refs), torch.cat(tols)


def _cta_ranges(tiles, sms):
    """[t_begin, t_end) of every CTA of stem_pool_kernel (grid = min(tiles, SMs), balanced contiguous ranges)."""
    grid = min(tiles, sms)
    per, rem = divmod(tiles, grid)
    return [(b * per + min(b, rem), (b + 1) * per + min(b + 1, rem)) for b in range(grid)]


# ===================================================================================================================
# 1. the staging buffer, bit for bit
# ===================================================================================================================
def _fp32_input(n, h, w, seed):
    """fp32 NCHW input whose fp16 values are disjoint from any normalised uint8 value (|x| >= 4), with values that
    round up to fp16 infinity, to the largest finite fp16, to subnormals and to -0."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(n, 3, h, w, generator=g) * 28 + 4) * torch.where(torch.rand(n, 3, h, w, generator=g) < 0.5, -1.0, 1.0)
    special = torch.tensor([65520.0, 65519.0, -65520.0, 2049.0, 2051.0, 6e-8, -1e-7, 3e-5, -0.0, 1e-9])
    x.view(-1)[:special.numel()] = special  # image 0, channel 0, first pixels
    return x


def _call_fused(L, N, x_dev, n, h, w, pad, w3, bias, relu, out, norm=None):
    if norm is None:
        N.check(L.ctl_stem_pool_fused(x_dev.data_ptr(), n, h, w, pad.data_ptr(), w3.data_ptr(), bias.data_ptr(), relu,
                                      out.data_ptr(), N.stream_ptr()))
    else:
        m, s = (C.c_float * 3)(*norm[0]), (C.c_float * 3)(*norm[1])
        N.check(L.ctl_stem_pool_fused_u8(x_dev.data_ptr(), n, h, w, m, s, pad.data_ptr(), w3.data_ptr(), bias.data_ptr(),
                                         relu, out.data_ptr(), N.stream_ptr()))


def _weights(seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(64, 3, 7, 7, generator=g) * 0.05, torch.randn(64, generator=g) * 0.1


def _check_staged(got, want, n, h, what):
    bad = got != want
    assert not bad.any(), (f"{what}: {int(bad.sum())} / {bad.numel()} fp16 of the staging buffer differ; first at "
                           f"{_where(int(bad.nonzero()[0]), n, h)}")


@gpu
@pytest.mark.parametrize("norm", ["imagenet", "odd"])
@pytest.mark.parametrize("h", [8, 12, 256])
@pytest.mark.parametrize("w", [8, 10, 62, 64, 126, 128])
def test_staging_buffer(w, h, norm):
    """fp32 entry, then the uint8 entry on the same buffer (as the handle does when forward and forward_u8 share a
    shape): each leaves exactly its own input in the interior and zeros everywhere else."""
    from ctl_b200.modelling.backbones.engine import pack_stem_fused

    N, L = _n()
    n = 2
    mean_std = IMAGENET if norm == "imagenet" else ODD_NORM
    seed = h * 1000 + w
    x = _fp32_input(n, h, w, seed)
    img = _crops(n, h, w, seed + 1)
    wt, b = _weights(seed)
    w3, bc = pack_stem_fused(wt.cuda()), b.cuda()
    pad = torch.zeros(L.ctl_stem_pad_bytes(n, h, w), dtype=torch.uint8, device="cuda")
    assert pad.numel() == 2 * (n * (h + 6) * WP * 4 + 128)
    hp, wp = _pool_shape(h, w)
    out = torch.full((n, hp, wp, 64), float("nan"), dtype=torch.float16, device="cuda")

    _call_fused(L, N, x.cuda(), n, h, w, pad, w3, bc, 0, out)
    torch.cuda.synchronize()
    _check_staged(pad.cpu().view(torch.int16), _staged(x.half()), n, h, "fp32 entry")

    want_u8 = _staged(_normalize_u8(img, *mean_std).half())
    _call_fused(L, N, img.cuda(), n, h, w, pad, w3, bc, 0, out, norm=mean_std)
    torch.cuda.synchronize()
    _check_staged(pad.cpu().view(torch.int16), want_u8, n, h, "uint8 entry after the fp32 entry")


# ===================================================================================================================
# 2. fused conv + pool against float64, per element
# ===================================================================================================================
def _grid_shape(target, sms):
    """(n, h) whose tile count n * h / 4 sits at (or, when no h in 8..64 divides it, next to) a multiple of the SM
    count: "two" (n = 1, h = 8); "sms-1" (< SMs: one tile per CTA, most starting inside an image); "sms"; "sms+1"
    (> SMs: the first CTA walks two tiles); "3sms+5" (uneven ranges of 3 and 4 tiles)."""
    if target == "two":
        return 1, 8
    want = {"sms-1": sms - 1, "sms": sms, "sms+1": sms + 1, "3sms+5": 3 * sms + 5}[target]
    ok = {"sms-1": lambda t: t < sms, "sms": lambda t: t == sms, "sms+1": lambda t: t > sms,
          "3sms+5": lambda t: t > 3 * sms}[target]
    best = None
    for hp in range(2, 17):
        for n in (want // hp, -(-want // hp)):
            t = n * hp
            if n < 1 or not ok(t):
                continue
            key = (abs(t - want), hp % 2 == 0, n)  # prefer odd row-pair counts: more ranges start inside an image
            if best is None or key < best[0]:
                best = (key, n, 4 * hp)
    assert best is not None, (target, sms)
    return best[1], best[2]


FUSED_CASES = [("width", 3, 16, w) for w in (8, 10, 62, 64, 126, 128)] + [("width", 2, 12, 10), ("width", 1, 8, 126)]
FUSED_CASES += [("grid", t, None, w) for t, w in (("two", 10), ("sms-1", 62), ("sms", 126), ("sms+1", 62),
                                                   ("3sms+5", 64))]
FUSED_CASES += [("shape", 3, 64, 48), ("shape", 2, 256, 128), ("shape", 40, 64, 32), ("shape", 5, 128, 64),
                ("shape", 1, 8, 8)]  # ranges that start inside an image and cross images at crop shapes


def _run_stem_case(n, h, w, relu, seed, sample=None, u8=False):
    from ctl_b200.modelling.backbones.engine import pack_stem_fused

    N, L = _n()
    img = _crops(n, h, w, seed)
    x = _normalize_u8(img, *IMAGENET)
    wt, b = _weights(seed + 7)
    w3, bc = pack_stem_fused(wt.cuda()), b.cuda()
    pad = torch.zeros(L.ctl_stem_pad_bytes(n, h, w), dtype=torch.uint8, device="cuda")
    hp, wp = _pool_shape(h, w)
    outs = []
    src = img.cuda() if u8 else x.cuda()
    for _ in range(2):
        out = torch.full((n, hp, wp, 64), float("nan"), dtype=torch.float16, device="cuda")
        _call_fused(L, N, src, n, h, w, pad, w3, bc, relu, out, norm=IMAGENET if u8 else None)
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), "two calls on the same input differ"
    buf = pad.cpu().view(torch.int16)
    x16 = _interior(buf, n, h, w)  # the input the kernel read (item 1 checks it is fp16(x))
    w16 = _unpack_w3(w3.cpu())
    assert not w16[:, 3].any() and not w16[..., 7].any()
    w16 = w16[:, :3, :, :7]
    sel = torch.arange(n) if sample is None else torch.tensor(sample)
    ref, tol = _stem_ref(x16[sel], w16, b, relu)
    got = outs[0].cpu()[sel].double().permute(0, 3, 1, 2)
    assert torch.isfinite(got).all(), "unwritten or non-finite outputs"
    err = (got - ref).abs()
    assert not (err > tol).any(), _report(err, tol) + " (index [sampled image, channel, row, column])"
    return float((err / tol).max())


@gpu
@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("kind,n,h,w", FUSED_CASES)
def test_stem_pool_fused(kind, n, h, w, relu):
    """Every width class at n = 3 (16 rows: 4 row pairs per image over 12 CTAs), the tile counts around the SM count
    and crop shapes; relu 0 (ResNet50's stem, all-negative windows occur) and 1 (IBN-a)."""
    if kind == "grid":
        n, h = _grid_shape(n, _sms())
    r = _run_stem_case(n, h, w, relu, seed=n * 10007 + h * 131 + w)
    print(f"fused stem {n}x{h}x{w} relu {relu}: max err/budget {r:.3f}")


@gpu
@pytest.mark.parametrize("n,h,w,relu,u8", [(256, 256, 128, 0, True), (128, 128, 64, 1, False)])
def test_stem_pool_fused_bench_batch(n, h, w, relu, u8):
    """The bench batch (256 x 256x128, ResNet50, from uint8 as forward_u8) and the IBN-a batch 128 x 128x64.  At
    256 x 256x128 the images checked are those of the whole ranges of CTAs 0, rem - 1, rem (the first with one tile
    fewer), the first CTA after 0 that starts at an image start, and the last CTA: every tile boundary of those
    ranges, with the recomputed row pair where a range starts inside an image.  At 128 x 128x64 every image."""
    sample = None
    if n == 256:
        hp = h // 4
        ranges = _cta_ranges(n * hp, _sms())
        rem = n * hp % len(ranges)
        at_image_start = [b for b in range(1, len(ranges)) if ranges[b][0] % hp == 0]
        pick = {0, max(rem - 1, 0), min(rem, len(ranges) - 1), len(ranges) - 1} | set(at_image_start[:1])
        sample = sorted({t // hp for b in pick for t in range(ranges[b][0], ranges[b][1])})
    r = _run_stem_case(n, h, w, relu, seed=n + h + w, sample=sample, u8=u8)
    print(f"fused stem {n}x{h}x{w} relu {relu}: images checked {sample or 'all'}; max err/budget {r:.3f}")


# ===================================================================================================================
# 3. the handle's stem and head folds on adversarial BatchNorm statistics
# ===================================================================================================================
GROUPS = ("var 0", "var 1e-7", "var 1e4", "negative gamma", "|mean| 30")
BN_KEYS = ("weight", "bias", "running_mean", "running_var")


def _adversarial_bn(c, seed, gain=1.0):
    """Eval BatchNorm of c channels, channel j in group GROUPS[j % 5]: running_var 0 or 1e-7 with gamma ~1e-2 (scale
    ~3.2 gain, and ~3.2 only because of eps), running_var 1e4 with gamma ~100, negative gamma, and |running_mean| 30
    with beta chosen in float64 so that beta - mean * scale is ~0.1.  The other statistics are gentle."""
    g = torch.Generator().manual_seed(seed)
    grp = torch.arange(c) % 5
    spread = 0.8 + 0.4 * torch.rand(c, generator=g)
    gamma = (0.5 + torch.rand(c, generator=g)) * gain
    var = 0.5 + torch.rand(c, generator=g)
    mean = 0.1 * torch.randn(c, generator=g)
    beta = 0.1 * torch.randn(c, generator=g)
    sign = torch.where(torch.rand(c, generator=g) < 0.5, -1.0, 1.0)
    gamma = torch.where(grp <= 1, 1e-2 * spread * gain, gamma)
    var = torch.where(grp == 0, 0.0, torch.where(grp == 1, 1e-7, var))
    gamma = torch.where(grp == 2, 100 * spread * gain, gamma)
    var = torch.where(grp == 2, 1e4, var)
    gamma = torch.where(grp == 3, -gamma, gamma)
    mean = torch.where(grp == 4, 30 * sign, mean)
    s = gamma.double() / torch.sqrt(var.double() + EPS)
    beta = torch.where(grp == 4, (mean.double() * s + 0.1 * torch.randn(c, generator=g).double()).float(), beta)
    return dict(weight=gamma, bias=beta, running_mean=mean, running_var=var)


def _put(sd, name, bn):
    for k in BN_KEYS:
        sd[f"{name}.{k}"] = bn[k]


def _get(sd, name):
    return {k: sd[f"{name}.{k}"] for k in BN_KEYS}


def _fold32(bn):
    """The fold of stem_pack_kernel / head_pack_kernel in torch fp32, every operation correctly rounded."""
    s = bn["weight"] / torch.sqrt(bn["running_var"] + EPS)
    return s, bn["bias"] - bn["running_mean"] * s


def _fold64(bn, how="right"):
    """float64 eval BatchNorm as scale and shift, or one of the plausible wrong folds."""
    g, beta, mean, var = (bn[k].double() for k in BN_KEYS)
    s = {"no_eps": lambda: g / torch.sqrt(var), "eps_outside": lambda: g / (torch.sqrt(var) + EPS)}.get(
        how, lambda: g / torch.sqrt(var + EPS))()
    return s, (beta + mean * s if how == "plus_mean" else beta - mean * s)


def _bn_stem_ref(x16, w, bn, relu, how="right"):
    """float64 maxpool(act(BN(conv(x16, w)))) on the unfolded fp32 weights, and its budget (module docstring)."""
    s, b = _fold64(bn, how)
    xd = x16.double()
    y = F.conv2d(xd, w.double(), None, 2, 3) * s[:, None, None] + b[:, None, None]
    mag = F.max_pool2d(F.conv2d(xd.abs(), (w.double() * s[:, None, None, None]).abs(), None, 2, 3), 3, 2, 1)
    ref = F.max_pool2d(y.clamp(min=0) if relu else y, 3, 2, 1)
    g, beta, mean, var = (bn[k].double() for k in BN_KEYS)
    tol = (2.0 ** -10 * F.max_pool2d(y.abs(), 3, 2, 1) + (2.0 ** -20 + 2.0 ** -11) * mag
           + 2.0 ** -22 * (beta.abs() + (mean * s).abs())[:, None, None])
    return ref, tol


def _head_ref(feat, bn, how="right"):
    s, b = _fold64(bn, how)
    f = feat.double()
    return f * s + b, 2.0 ** -21 * ((f * s).abs() + (bn["running_mean"].double() * s).abs() + bn["bias"].double().abs())


HANDLES = {"r50": ("bottleneck", False, O.R50_LAYERS), "r50_ibn": ("bottleneck", True, O.R50_LAYERS),
           "r18": ("basic", False, BO.BASIC_LAYERS["resnet18"])}


@pytest.fixture(scope="module")
def engines():
    cache = {}

    def get(arch):
        if arch not in cache:
            from ctl_b200.modelling.backbones.engine import TrunkEngine

            block, ibn, layers = HANDLES[arch]
            sd = BO.make_trunk_state(seed=3, layers=layers) if block == "basic" else O.make_trunk_state(seed=3, ibn=ibn)
            _put(sd, "bn1", _adversarial_bn(64, seed=17))
            head = _adversarial_bn(512 if block == "basic" else 2048, seed=19)
            cache[arch] = (TrunkEngine(sd, "cuda", ibn=ibn, layers=layers, bn_head=head, block=block), sd, head)
        return cache[arch]

    yield get
    cache.clear()


STEM_ROUTES = [(2, 256, 128, "fp32"), (2, 256, 128, "u8"), (2, 64, 32, "fp32"), (2, 64, 32, "u8"), (2, 64, 126, "fp32"),
               (2, 64, 126, "u8"),
               (1, 320, 320, "fp32"),  # wider than the fused stem takes: tensor-core stem + max-pool
               (2, 254, 128, "fp32")]  # h % 4 == 2: the tensor-core route at w <= 128


@gpu
@pytest.mark.parametrize("n,h,w,src", STEM_ROUTES)
@pytest.mark.parametrize("arch", list(HANDLES))
def test_handle_stem_fold(engines, arch, n, h, w, src):
    """(a) teacher-forced: against the fold recomputed in torch fp32 (s = g / sqrt(v + eps), b = beta - mean s,
    fp16(w s)), the budget of item 2; (b) against float64 BN(conv(x16, w)) on the unfolded weights."""
    N, L = _n()
    eng, sd, _ = engines(arch)
    relu = int(eng.ibn)
    img = _crops(n, h, w, seed=h * 7 + w + n)
    x = _normalize_u8(img, *IMAGENET)
    hp, wp = _pool_shape(h, w)
    out = torch.full((n, hp, wp, 64), float("nan"), dtype=torch.float16, device="cuda")
    ws = eng._workspace(n, h, w)
    xin = img.cuda() if src == "u8" else x.cuda()
    norm = [(C.c_float * 3)(*v) for v in IMAGENET] if src == "u8" else [None, None]
    N.check(L.ctl_embed_stem(eng._h, xin.data_ptr(), n, h, w, norm[0], norm[1], out.data_ptr(), ws.data_ptr(), ws.numel(),
                             N.stream_ptr()))
    torch.cuda.synchronize()
    got = out.cpu().double().permute(0, 3, 1, 2)
    assert torch.isfinite(got).all(), "unwritten or non-finite outputs"
    x16, wt, bn = x.half(), sd["conv1.weight"], _get(sd, "bn1")
    s32, b32 = _fold32(bn)
    ref, tol = _stem_ref(x16, (wt * s32[:, None, None, None]).half(), b32, relu)
    err = (got - ref).abs()
    assert not (err > tol).any(), "teacher-forced fold: " + _report(err, tol)
    ra = float((err / tol).max())
    ref, tol = _bn_stem_ref(x16, wt, bn, relu)
    err = (got - ref).abs()
    assert not (err > tol).any(), "float64 BatchNorm: " + _report(err, tol)
    print(f"{arch} stem {n}x{h}x{w} {src}: max err/budget (a) {ra:.3f}, (b) {float((err / tol).max()):.3f}")


@gpu
@pytest.mark.parametrize("arch", list(HANDLES))
def test_handle_head_fold(engines, arch):
    """emb == float64 F.batch_norm of the device's own feat, per element (feat itself is test_eval_kernels_gpu.py's)."""
    N, L = _n()
    eng, _, head = engines(arch)
    n, hw, c = 4, 32, eng.feature_dim
    g = torch.Generator().manual_seed(c)
    a = (torch.randn(n, hw, c, generator=g) * 2 + torch.randn(c, generator=g)).half().cuda()
    feat = torch.full((n, c), float("nan"), device="cuda")
    emb = torch.full((n, c), float("nan"), device="cuda")
    N.check(L.ctl_embed_head(eng._h, a.data_ptr(), n, hw, feat.data_ptr(), emb.data_ptr(), N.stream_ptr()))
    torch.cuda.synchronize()
    feat, emb = feat.cpu(), emb.cpu()
    assert torch.isfinite(feat).all() and torch.isfinite(emb).all(), "unwritten or non-finite outputs"
    ref = F.batch_norm(feat.double(), head["running_mean"].double(), head["running_var"].double(),
                       head["weight"].double(), head["bias"].double(), False, 0.0, EPS)
    _, tol = _head_ref(feat, head)
    err = (emb.double() - ref).abs()
    assert not (err > tol).any(), _report(err, tol)
    print(f"{arch} head: max err/budget {float((err / tol).max()):.3f}")


# ===================================================================================================================
# 4. block folds through the whole trunk
# ===================================================================================================================
TRUNKS = {"r18": ("basic", False, BO.BASIC_LAYERS["resnet18"], ".bn2"),
          "r50_ibn": ("bottleneck", True, O.R50_LAYERS, ".bn3")}


def _adversarial_state(arch, seed=23):
    """Adversarial statistics in every BatchNorm.  Main-path BNs get gain 1/2 (the scale's rms over the five groups is
    then ~1), residual-branch BNs (bn3 / bn2, as make_trunk_state's small bn3) 1/8, so that activations stay O(1)."""
    block, ibn, layers, branch = TRUNKS[arch]
    sd = BO.make_trunk_state(seed=seed, layers=layers) if block == "basic" else O.make_trunk_state(seed=seed, ibn=ibn)
    names = [k[:-len(".running_var")] for k in sd if k.endswith(".running_var")]
    for i, name in enumerate(names):
        _put(sd, name, _adversarial_bn(sd[name + ".running_var"].numel(), seed * 1000 + i,
                                       0.125 if name.endswith(branch) else 0.5))
    return sd


def _trunk_sim(arch, x, sd):
    block, ibn, layers, _ = TRUNKS[arch]
    with torch.no_grad():
        if block == "basic":
            return BO.trunk_forward_fp16sim(x, sd, layers=layers)[1]
        return O.trunk_forward_fp16sim(x, sd, ibn=ibn, layers=layers)[1]


def _trunk_input():
    return _normalize_u8(_crops(2, 128, 64, seed=29), *IMAGENET)


@gpu
@pytest.mark.parametrize("arch", list(TRUNKS))
def test_trunk_adversarial_folds(arch):
    """ResNet18 (downsample blocks through ctl_conv3x3_dual) and ResNet50-IBN-a (the dual 1x1, the IBN BatchNorm on
    channels [half, C)) with adversarial statistics in every BatchNorm, against the fp16-rounding checkers."""
    from ctl_b200.modelling.backbones.engine import TrunkEngine

    block, ibn, layers, _ = TRUNKS[arch]
    sd = _adversarial_state(arch)
    x = _trunk_input()
    feat = TrunkEngine(sd, "cuda", ibn=ibn, layers=layers, block=block).forward(x.cuda())["global_feat"].cpu()
    sim = _trunk_sim(arch, x, sd)
    assert torch.isfinite(feat).all()
    scale = float(sim.abs().max())
    err = (feat - sim).abs()
    tol = torch.full_like(err, 3e-3 * scale)
    assert not (err > tol).any(), _report(err, tol)
    print(f"{arch} trunk: |feat|max {scale:.4f}; max err/budget {float((err / tol).max()):.3f}")


# ===================================================================================================================
# 5. CPU self-checks of the models and references above
# ===================================================================================================================
@pytest.mark.parametrize("n,h,w", [(2, 12, 10), (1, 16, 64), (1, 8, 126), (2, 20, 128)])
def test_staging_and_operand_model_is_the_convolution(n, h, w):
    """The staging layout and the [28][64][8] operand, read back as the kernel's windows read them, are F.conv2d
    (7x7 / 2, pad 3) of fp16(x) and fp16(w) in float64; the interior read-back is the input."""
    from ctl_b200.modelling.backbones.engine import pack_stem_fused

    x16 = _normalize_u8(_crops(n, h, w, seed=h + w), *IMAGENET).half()
    wt, _ = _weights(h * w)
    buf, w3 = _staged(x16), pack_stem_fused(wt)
    assert torch.equal(_bits(_interior(buf, n, h, w)), _bits(x16))
    unpacked = _unpack_w3(w3)
    assert not unpacked[:, 3].any() and not unpacked[..., 7].any()
    assert torch.equal(_bits(unpacked[:, :3, :, :7].contiguous()), _bits(wt.half()))
    got = _conv_as_read(buf, w3, n, h, w)
    ref = F.conv2d(x16.double(), wt.half().double(), None, 2, 3)
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)


def test_odd_norm_separates_division_from_reciprocal():
    """With ODD_NORM, (u / 255 - m) / s and (u / 255 - m) * (1 / s) round to different fp16 for a u of KEY_U8 in
    every channel, so item 1 sees a packing kernel that multiplies by a reciprocal."""
    u = np.asarray(KEY_U8, np.float32) / np.float32(255)
    for m, s in zip(*ODD_NORM):
        m, s = np.float32(m), np.float32(s)
        div = ((u - m) / s).astype(np.float16)
        rcp = ((u - m) * (np.float32(1) / s)).astype(np.float16)
        assert (div.view(np.int16) != rcp.view(np.int16)).any(), (m, s)


def _change(wrong, right, tol):
    """max |wrong - right| / tol; a non-finite wrong result counts as infinitely far."""
    if not torch.isfinite(wrong).all():
        return math.inf
    return float(((wrong - right).abs() / tol).max())


@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("how", ["no_eps", "eps_outside", "plus_mean"])
def test_wrong_stem_and_head_folds_exceed_tolerance(how, relu):
    """Each wrong fold moves the float64 stem reference of item 3 (b) and the head reference by >= 10x the budgets."""
    x16 = _normalize_u8(_crops(2, 32, 32, seed=1), *IMAGENET).half()
    bn = _adversarial_bn(64, seed=17)
    wt = O.make_trunk_state(seed=3)["conv1.weight"]
    right, tol = _bn_stem_ref(x16, wt, bn, relu)
    wrong, _ = _bn_stem_ref(x16, wt, bn, relu, how)
    assert _change(wrong, right, tol) >= 10
    feat = torch.randn(4, 2048, generator=torch.Generator().manual_seed(2)) * 2
    head = _adversarial_bn(2048, seed=19)
    right, tol = _head_ref(feat, head)
    wrong, _ = _head_ref(feat, head, how)
    assert _change(wrong, right, tol) >= 10


def _refold(sd, name, s, b):
    """Re-expresses BatchNorm `name` as the given scale and shift (float64), which fold to them within fp32 rounding."""
    _put(sd, name, dict(weight=(s * math.sqrt(1 + EPS)).float(), bias=b.float(), running_mean=torch.zeros_like(b).float(),
                        running_var=torch.ones_like(b).float()))


def _wrong_state(sd, how):
    out = dict(sd)
    for name in [k[:-len(".running_var")] for k in sd if k.endswith(".running_var")]:
        bn = _get(sd, name)
        if how in ("no_eps", "eps_outside", "plus_mean"):
            _refold(out, name, *_fold64(bn, how))
        elif how == "dual_bias_dropped" and name.endswith("downsample.1"):
            s, _ = _fold64(bn)
            _refold(out, name, s, torch.zeros_like(s))
        elif how == "ibn_offset" and name.endswith("bn1.BN"):
            # folded at channel offset 0: channels [half, C) keep the raw convolution, and the InstanceNorm that
            # follows channels [0, half) cancels the fold there but for its sign
            s, _ = _fold64(bn)
            _refold(out, name, torch.ones_like(s), torch.zeros_like(s))
            iw = name[:-len(".BN")] + ".IN.weight"
            out[iw] = sd[iw] * torch.sign(s).float()
    return out


@pytest.mark.parametrize("arch,how", [(a, h) for a in TRUNKS for h in ("no_eps", "eps_outside", "plus_mean",
                                                                        "dual_bias_dropped")] + [("r50_ibn", "ibn_offset")])
def test_wrong_trunk_folds_exceed_tolerance(arch, how):
    """Each wrong block fold moves the item 4 checker's features by >= 10x its 3e-3 * scale bound; the right one
    keeps the activations finite and O(1) in fp16."""
    sd, x = _adversarial_state(arch), _trunk_input()
    right = _trunk_sim(arch, x, sd)
    scale = float(right.abs().max())
    assert torch.isfinite(right).all() and 0.05 < scale < 100, scale
    wrong = _trunk_sim(arch, x, _wrong_state(sd, how))
    assert _change(wrong, right, torch.full_like(right, 3e-3 * scale)) >= 10
