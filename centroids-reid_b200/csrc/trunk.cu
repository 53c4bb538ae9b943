// Whole-trunk entry points of the C ABI (SURVEY 8b: ctl_weights_pack + ctl_embed_forward): the layer graph of the eval
// embedding path -- ResNet.forward / ResNet_IBN.forward (modelling/backbones/resnet.py:122-133, resnet_ibn_a.py:126-141)
// over Bottleneck (ResNet50/101/152, -IBN-a) or BasicBlock (ResNet18/34) blocks,
// Baseline.forward's global average pool (modelling/baseline.py:91-96) and the eval BatchNorm1d of
// ModelBase.validation_step (modelling/bases.py:169-177) -- behind an opaque handle.  This is the eval trunk's only
// driver: modelling/backbones/engine.py::TrunkEngine is its ctypes form, and a host that is not Python binds the same calls.
//
// The handle owns the PACKED operands: [Cout][kh][kw][Cin] fp16 weights with the eval BatchNorm folded in and fp32
// biases, produced on the device from the reference's fp32 state_dict tensors (fold_pack_kernel: fp32 divide / sqrt /
// multiply / subtract, each correctly rounded, then one rounding to fp16), the K-concatenated [W3 | Wd] (bottleneck) or
// [W2 | Wd] (BasicBlock) matrices of every block with a downsample, the two stem layouts, and one zero-bordered staging buffer of the fused stem per input shape.
// Activations live in a caller-provided workspace.
#include <math.h>
#include <string.h>

#include <array>
#include <map>
#include <string>
#include <vector>

#include "common.h"
#include "resnet.h"
#include "wgmma.cuh"

namespace ctl {

// w [cout][cin][k][k] fp32 (+ BatchNorm gamma/beta/mean/var of `nbn` channels starting at channel c0; nullptr = no fold)
//   -> out [cout][k][k][cin] fp16 rows of pitch `pitch` elements at column offset `col0`;
//   bias[c] (= beta - mean * scale) written, or ADDED when `accumulate` (the [W3 | Wd] pair shares one bias vector).
__global__ void fold_pack_kernel(const float* __restrict__ w, int cout, int cin, int k, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, const float* __restrict__ mean,
                                 const float* __restrict__ var, int c0, __half* __restrict__ out, long long pitch, int col0,
                                 float* __restrict__ bias, int accumulate) {
  const int co = blockIdx.x;
  float scale = 1.f, b = 0.f;
  if (gamma != nullptr && co >= c0) {
    const int j = co - c0;
    scale = __fdiv_rn(gamma[j], __fsqrt_rn(__fadd_rn(var[j], BN_EPS)));
    b = __fsub_rn(beta[j], __fmul_rn(mean[j], scale));
  }
  const int kk = k * k;
  for (int i = threadIdx.x; i < cin * kk; i += blockDim.x) {
    const int ci = i % cin, rs = i / cin;  // output order (r, s, ci)
    const float v = w[((size_t)co * cin + ci) * kk + rs];
    out[(size_t)co * pitch + col0 + (size_t)rs * cin + ci] = __float2half_rn(__fmul_rn(v, scale));
  }
  if (threadIdx.x == 0 && bias != nullptr) bias[co] = accumulate ? __fadd_rn(bias[co], b) : b;
}

// stem layouts (ctl_stem_conv7x7_tc: [64][192], k = (c*7 + r)*8 + s, s = 7 and k >= 168 zero;  ctl_stem_pool_fused:
// [28][64][8], chunk = r*4 + s/2, element = (s%2)*4 + ch, ch == 3 and s == 7 zero) -- see stem_pack
__global__ void stem_pack_kernel(const float* __restrict__ w, const float* __restrict__ gamma, const float* __restrict__ beta,
                                 const float* __restrict__ mean, const float* __restrict__ var, __half* __restrict__ w192,
                                 __half* __restrict__ w3, float* __restrict__ bias) {
  const int o = blockIdx.x;
  float scale = 1.f;
  if (gamma != nullptr) {
    scale = __fdiv_rn(gamma[o], __fsqrt_rn(__fadd_rn(var[o], BN_EPS)));
    if (threadIdx.x == 0) bias[o] = __fsub_rn(beta[o], __fmul_rn(mean[o], scale));
  }
  for (int i = threadIdx.x; i < 192; i += blockDim.x) {
    float v = 0.f;
    if (i < 168) {
      const int cr = i / 8, s = i % 8;
      if (s < 7) v = __fmul_rn(w[(size_t)o * 147 + cr * 7 + s], scale);
    }
    w192[(size_t)o * 192 + i] = __float2half_rn(v);
  }
  if (w3 == nullptr) return;
  for (int i = threadIdx.x; i < 28 * 8; i += blockDim.x) {
    const int chunk = i / 8, e = i % 8, r = chunk / 4, s = (chunk % 4) * 2 + e / 4, ch = e % 4;
    float v = 0.f;
    if (s < 7 && ch < 3) v = __fmul_rn(w[(size_t)o * 147 + (ch * 7 + r) * 7 + s], scale);
    w3[((size_t)chunk * 64 + o) * 8 + e] = __float2half_rn(v);
  }
}

int stem_pack(const float* w, const float* gamma, const float* beta, const float* mean, const float* var, __half* w192,
              __half* w3, float* bias, cudaStream_t st) {
  stem_pack_kernel<<<64, 128, 0, st>>>(w, gamma, beta, mean, var, w192, w3, bias);
  CTL_LAUNCH_CHECK();
  return 0;
}

__global__ void head_pack_kernel(const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ mean,
                                 const float* __restrict__ var, int n, float* __restrict__ scale, float* __restrict__ shift) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float s = __fdiv_rn(gamma[i], __fsqrt_rn(__fadd_rn(var[i], BN_EPS)));
  scale[i] = s;
  shift[i] = __fsub_rn(beta[i], __fmul_rn(mean[i], s));
}

// a convolution of the layout and its packed operands: folded fp16 weights w, fp32 biases b
struct PackedConv : ConvLayout {
  __half* w = nullptr;
  float* b = nullptr;
};
struct TrunkBlock : BlockLayout<PackedConv> {
  float *in_gamma = nullptr, *in_beta = nullptr;  // c1's InstanceNorm (IBN-a)
  __half* dual_w = nullptr;
  float* dual_b = nullptr;
};

}  // namespace ctl

struct ctl_trunk {
  int block = CTL_BLOCK_BOTTLENECK, feature_dim = 2048;
  int ibn = 0;
  bool packed = false, has_head = false;
  std::vector<ctl::TrunkBlock> blocks;
  __half *stem_w192 = nullptr, *stem_w3 = nullptr;
  float* stem_b = nullptr;
  float *head_scale = nullptr, *head_shift = nullptr;
  // (n, h, w) -> zero-bordered staging buffer of the fused stem.  Kept until ctl_trunk_destroy: a CUDA graph captured at
  // one shape still reads its buffer after calls at other shapes.
  std::map<std::array<int, 3>, void*> stem_pads;
  int32_t launches = 0;      // kernels launched by the last ctl_embed_* call
  std::vector<void*> owned;  // every cudaMalloc of this handle
};

namespace ctl {

// packs `c` with its BatchNorm folded in (IBN-a: channels [in_half, cout) only)
static int pack_conv(ctl_trunk* h, const NamedMap& m, PackedConv& c, cudaStream_t st) {
  int rc = 0;
  const float* w = lookup(m, c.conv + ".weight", (long long)c.cout * c.cin * c.k * c.k, &rc);
  if (rc) return rc;
  const int nbn = c.cout - c.in_half;
  const float *g = lookup(m, c.bn + ".weight", nbn, &rc), *b = lookup(m, c.bn + ".bias", nbn, &rc),
              *mu = lookup(m, c.bn + ".running_mean", nbn, &rc), *va = lookup(m, c.bn + ".running_var", nbn, &rc);
  if (rc) return rc;
  if (!c.w) c.w = dev_alloc<__half>(h, (size_t)c.cout * c.cin * c.k * c.k);
  if (!c.b) c.b = dev_alloc<float>(h, c.cout);
  if (!c.w || !c.b) {
    set_error("ctl_weights_pack: out of device memory");
    return (int)cudaErrorMemoryAllocation;
  }
  fold_pack_kernel<<<c.cout, 256, 0, st>>>(w, c.cout, c.cin, c.k, g, b, mu, va, c.in_half, c.w, (long long)c.cin * c.k * c.k, 0,
                                           c.b, 0);
  CTL_LAUNCH_CHECK();
  return 0;
}

// The single-GEMM form of the last convolution `last` of `blk` (conv3 of a bottleneck, conv2 of a BasicBlock) + its
// downsample: [W_last | Wd] with bias_last + bias_d (ctl_conv1x1_dual_nhwc_f16 / ctl_conv3x3_dual_nhwc_f16).  `last` and
// the downsample must be packed already.
static int pack_dual(ctl_trunk* h, const NamedMap& m, TrunkBlock& blk, const PackedConv& last, cudaStream_t st) {
  int rc = 0;
  const PackedConv& d = blk.down;
  const int km = last.k * last.k * last.cin;  // row length of the packed [cout][k][k][cin] weights
  const int kt = km + d.cin;
  if (!blk.dual_w) {
    blk.dual_w = dev_alloc<__half>(h, (size_t)last.cout * kt);
    blk.dual_b = dev_alloc<float>(h, last.cout);
  }
  if (!blk.dual_w || !blk.dual_b) {
    set_error("ctl_weights_pack: out of device memory");
    return (int)cudaErrorMemoryAllocation;
  }
  CTL_CUDA(cudaMemcpy2DAsync(blk.dual_w, (size_t)kt * 2, last.w, (size_t)km * 2, (size_t)km * 2, last.cout,
                             cudaMemcpyDeviceToDevice, st));
  CTL_CUDA(cudaMemcpy2DAsync(blk.dual_w + km, (size_t)kt * 2, d.w, (size_t)d.cin * 2, (size_t)d.cin * 2, last.cout,
                             cudaMemcpyDeviceToDevice, st));
  // bias_last + bias_d, one fp32 add per channel
  CTL_CUDA(cudaMemcpyAsync(blk.dual_b, last.b, last.cout * sizeof(float), cudaMemcpyDeviceToDevice, st));
  fold_pack_kernel<<<last.cout, 32, 0, st>>>(lookup(m, d.conv + ".weight", (long long)d.cout * d.cin, &rc), d.cout, 0, 1,
                                             lookup(m, d.bn + ".weight", d.cout, &rc), lookup(m, d.bn + ".bias", d.cout, &rc),
                                             lookup(m, d.bn + ".running_mean", d.cout, &rc),
                                             lookup(m, d.bn + ".running_var", d.cout, &rc), 0, d.w, 0, 0, blk.dual_b, 1);
  CTL_LAUNCH_CHECK();
  return rc;
}

}  // namespace ctl

using namespace ctl;

extern "C" {

int ctl_trunk_create(ctl_trunk** out, int32_t block, int32_t ibn, int32_t last_stride, const int32_t stage_blocks[4]) {
  CTL_CHECK_ARG(out != nullptr, "null pointer");
  ctl_trunk* h = new ctl_trunk();
  if (int rc = resnet_layout(block, ibn, last_stride, stage_blocks, &h->feature_dim, &h->blocks)) {
    delete h;
    return rc;
  }
  h->block = block;
  h->ibn = ibn ? 1 : 0;
  *out = h;
  return 0;
}

int32_t ctl_trunk_feature_dim(const ctl_trunk* h) { return h ? h->feature_dim : 0; }

void ctl_trunk_destroy(ctl_trunk* h) {
  if (!h) return;
  for (void* p : h->owned) cudaFree(p);
  delete h;
}

int ctl_weights_pack(ctl_trunk* h, const ctl_named_tensor* tensors, int32_t n_tensors, ctl_stream_t stream) {
  CTL_CHECK_ARG(h && tensors && n_tensors > 0, "bad arguments");
  int rc = ctl_device_check();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  NamedMap m;
  if ((rc = index_named(tensors, n_tensors, "ctl_weights_pack", "tensor", &m))) return rc;
  // ---- stem ----
  {
    const float* w = lookup(m, "conv1.weight", 64 * 147, &rc);
    const float *g = lookup(m, "bn1.weight", 64, &rc), *b = lookup(m, "bn1.bias", 64, &rc),
                *mu = lookup(m, "bn1.running_mean", 64, &rc), *va = lookup(m, "bn1.running_var", 64, &rc);
    if (rc) return rc;
    if (!h->stem_w192) {
      h->stem_w192 = dev_alloc<__half>(h, 64 * 192);
      h->stem_w3 = dev_alloc<__half>(h, 28 * 64 * 8);
      h->stem_b = dev_alloc<float>(h, 64);
    }
    if (!h->stem_w192 || !h->stem_w3 || !h->stem_b) {
      set_error("ctl_weights_pack: out of device memory");
      return (int)cudaErrorMemoryAllocation;
    }
    if ((rc = stem_pack(w, g, b, mu, va, h->stem_w192, h->stem_w3, h->stem_b, st))) return rc;
  }
  // ---- blocks ----
  for (TrunkBlock& blk : h->blocks) {
    for (PackedConv* c : blk.state_dict_order()) {
      if (!c) continue;
      if ((rc = pack_conv(h, m, *c, st))) return rc;
      if (!c->in_half) continue;
      // IBN: channels [0, half) keep the raw convolution, and InstanceNorm + ReLU follow as their own kernel
      const float *ig = lookup(m, c->in + ".weight", c->in_half, &rc), *ib = lookup(m, c->in + ".bias", c->in_half, &rc);
      if (rc) return rc;
      if (!blk.in_gamma) {
        blk.in_gamma = dev_alloc<float>(h, c->in_half);
        blk.in_beta = dev_alloc<float>(h, c->in_half);
      }
      CTL_CUDA(cudaMemcpyAsync(blk.in_gamma, ig, c->in_half * sizeof(float), cudaMemcpyDeviceToDevice, st));
      CTL_CUDA(cudaMemcpyAsync(blk.in_beta, ib, c->in_half * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    if (blk.has_down && (rc = pack_dual(h, m, blk, blk.bottleneck ? blk.c3 : blk.c2, st))) return rc;
  }
  // ---- optional BatchNorm1d head (ModelBase.bn, modelling/bases.py:83) ----
  h->has_head = m.refs.count("bn_head.weight") != 0;
  if (h->has_head) {
    const int fd = h->feature_dim;
    const float *g = lookup(m, "bn_head.weight", fd, &rc), *b = lookup(m, "bn_head.bias", fd, &rc),
                *mu = lookup(m, "bn_head.running_mean", fd, &rc), *va = lookup(m, "bn_head.running_var", fd, &rc);
    if (rc) return rc;
    if (!h->head_scale) {
      h->head_scale = dev_alloc<float>(h, fd);
      h->head_shift = dev_alloc<float>(h, fd);
    }
    head_pack_kernel<<<(fd + 255) / 256, 256, 0, st>>>(g, b, mu, va, fd, h->head_scale, h->head_shift);
    CTL_LAUNCH_CHECK();
  }
  h->packed = true;
  return 0;
}

}  // extern "C"

namespace ctl {

static size_t round256(size_t b) { return (b + 255) & ~(size_t)255; }
static bool fused_stem_fits(int hgt, int wid) { return hgt % 4 == 0 && wid % 2 == 0 && wid <= 128; }

// One of the activation slots of the block walk on a [n, hp, wp, 64] stem output: layer1's output is the largest tensor
// the blocks write (each later stage halves both sides -- stride-2 convolutions take even sides only -- before it
// doubles the channels), [n, hp, wp, 256] for bottlenecks and [n, hp, wp, 64] for BasicBlocks.
static size_t block_slot_bytes(const ctl_trunk* h, int n, int hp, int wp) {
  return round256((size_t)n * hp * wp * (h->block == CTL_BLOCK_BASIC ? 64 : 256) * 2);
}
// the bottleneck walk rotates five slots, the BasicBlock walk three (block input, conv1 output, block output)
static int block_slots(const ctl_trunk* h) { return h->block == CTL_BLOCK_BASIC ? 3 : 5; }
// the tensor-core stem's conv output [n, h/2, w/2, 64], which is larger than a slot when h/2 or w/2 is odd
static size_t stem_tmp_bytes(int n, int hgt, int wid) { return round256((size_t)n * stem_side(hgt) * stem_side(wid) * 64 * 2); }

static int check_workspace(size_t need, size_t have) {
  if (have < need) {
    set_error("workspace too small: need %zu bytes, have %zu", need, have);
    return CTL_ERR_WORKSPACE;
  }
  return 0;
}

// what every ctl_embed_* call checks once its arguments are valid
static int begin_call(ctl_trunk* h) {
  CTL_CHECK_ARG(h->packed, "ctl_weights_pack has not been called on this handle");
  h->launches = 0;
  return ctl_device_check();
}

static int stem_pad(ctl_trunk* h, int n, int hgt, int wid, cudaStream_t st, void** pad) {
  const std::array<int, 3> key = {n, hgt, wid};
  auto it = h->stem_pads.find(key);
  if (it != h->stem_pads.end()) {
    *pad = it->second;
    return 0;
  }
  cudaStreamCaptureStatus capture;
  CTL_CUDA(cudaStreamIsCapturing(st, &capture));
  CTL_CHECK_ARG(capture == cudaStreamCaptureStatusNone,
                "the fused stem's staging buffer for n=%d, %dx%d would be allocated during stream capture: run one call "
                "at this shape on the handle before capturing",
                n, hgt, wid);
  const size_t bytes = ctl_stem_pad_bytes(n, hgt, wid);
  void* p = dev_alloc<char>(h, bytes);
  if (!p) {
    set_error("out of device memory (stem staging buffer of %zu bytes)", bytes);
    return (int)cudaErrorMemoryAllocation;
  }
  CTL_CUDA(cudaMemsetAsync(p, 0, bytes, st));  // the zero border is written once
  h->stem_pads[key] = p;
  *pad = p;
  return 0;
}

// conv1 + bn1 (+ReLU for IBN-a) + maxpool -> out [n, hp, wp, 64]; x is fp32 NCHW, or uint8 NHWC when mean3 / std3 are
// given (fused stem only).  The tensor-core stem's conv output goes to `tmp` (stem_tmp_bytes).
static int run_stem(ctl_trunk* h, const void* x, const float* mean3, const float* std3, int n, int hgt, int wid, void* out,
                    void* tmp, cudaStream_t st) {
  int rc;
  h->launches += 2;  // input packing + conv/pool, or conv + pool
  if (fused_stem_fits(hgt, wid)) {
    void* pad = nullptr;
    if ((rc = stem_pad(h, n, hgt, wid, st, &pad))) return rc;
    return mean3 ? ctl_stem_pool_fused_u8(x, n, hgt, wid, mean3, std3, pad, h->stem_w3, h->stem_b, h->ibn, out, st)
                 : ctl_stem_pool_fused(static_cast<const float*>(x), n, hgt, wid, pad, h->stem_w3, h->stem_b, h->ibn, out, st);
  }
  if ((rc = ctl_stem_conv7x7_tc(static_cast<const float*>(x), n, hgt, wid, h->stem_w192, h->stem_b, h->ibn, tmp, st))) return rc;
  return ctl_maxpool3x3s2_nhwc_f16(tmp, n, stem_side(hgt), stem_side(wid), 64, out, st);
}

static int run_conv(ctl_trunk* h, const PackedConv& c, const void* x, int n, int hh, int ww, const void* residual, void* out,
                    cudaStream_t st) {
  ++h->launches;
  return ctl_conv2d_nhwc_f16(x, n, hh, ww, c.cin, c.w, c.b, residual, out, c.cout, c.k, c.stride, c.relu, c.in_half, st);
}

// The bottleneck walk on x [n, hh, ww, 64].  Intermediates rotate through five workspace slots of `slot` bytes; x is
// slot x_slot (recycled once read) or, with x_slot < 0, a caller tensor that is never written.  The last block writes
// `out` when it is given, else a slot.  *y = the trunk output [n, *hh, *ww, 2048].
static int run_blocks(ctl_trunk* h, const void* x, int x_slot, int n, int* hh, int* ww, char* ws, size_t slot, void* out,
                      const void** y, cudaStream_t st) {
  int rc;
  void* const buf[5] = {ws, ws + slot, ws + 2 * slot, ws + 3 * slot, ws + 4 * slot};
  const void* a = x;
  int cur = x_slot;   // slot holding the block input; < 0: the caller's tensor
  int o1_ready = -1;  // slot holding this block's conv1 output when the previous block's launch computed it
  for (size_t bi = 0; bi < h->blocks.size(); ++bi) {
    const TrunkBlock& blk = h->blocks[bi];
    // roles of four slots other than the input's; a conv1 output computed ahead keeps its slot (dead again once conv2
    // has read it, so the next chained launch writes there too) and the other roles rotate around it
    int role[4], k = 0;
    if (o1_ready >= 0) role[k++] = o1_ready;
    for (int i = 1; i <= 5 && k < 4; ++i)
      if ((cur + i) % 5 != cur && (cur + i) % 5 != o1_ready) role[k++] = (cur + i) % 5;
    void* o1 = buf[role[0]];
    void* o2 = buf[role[1]];
    void* res = buf[role[2]];
    void* dst = out && bi + 1 == h->blocks.size() ? out : buf[role[3]];
    const int h1 = *hh, w1 = *ww;
    if (o1_ready < 0 && (rc = run_conv(h, blk.c1, a, n, h1, w1, nullptr, o1, st))) return rc;
    if (blk.c1.in_half) {
      ++h->launches;
      if ((rc = ctl_instnorm_relu_nhwc_f16(o1, n, h1 * w1, blk.c1.cout, blk.c1.in_half, blk.in_gamma, blk.in_beta, BN_EPS, st)))
        return rc;
    }
    const int s = blk.c2.stride;
    const int h2 = (h1 + 2 - 3) / s + 1, w2 = (w1 + 2 - 3) / s + 1;
    if ((rc = run_conv(h, blk.c2, o1, n, h1, w1, nullptr, o2, st))) return rc;
    const bool dual = blk.has_down && h1 % s == 0 && w1 % s == 0;
    const void* r = a;
    if (blk.has_down && !dual) {
      if ((rc = run_conv(h, blk.down, a, n, h1, w1, nullptr, res, st))) return rc;
      r = res;
    }
    // the next block's conv1 in this launch's epilogue: its output goes to o1's slot (a and res are still read)
    const PackedConv* nx = bi + 1 < h->blocks.size() ? &h->blocks[bi + 1].c1 : nullptr;
    const bool chain = nx && ctl_conv1x1_chain_supported(blk.c3.cout, nx->cout);
    if (chain || dual) ++h->launches;  // run_conv counts the plain conv3
    if (chain) {
      if (dual)
        rc = ctl_conv1x1_chain_nhwc_f16(o2, blk.c3.cin, a, h1, w1, blk.down.cin, s, n, blk.dual_w, blk.dual_b, nullptr, dst,
                                        blk.c3.cout, nx->w, nx->b, nx->cout, nx->in_half, o1, st);
      else
        rc = ctl_conv1x1_chain_nhwc_f16(o2, blk.c3.cin, nullptr, h2, w2, 0, 1, n, blk.c3.w, blk.c3.b, r, dst, blk.c3.cout,
                                        nx->w, nx->b, nx->cout, nx->in_half, o1, st);
    } else if (dual) {
      rc = ctl_conv1x1_dual_nhwc_f16(o2, blk.c3.cin, a, h1, w1, blk.down.cin, s, n, blk.dual_w, blk.dual_b, dst, blk.c3.cout, 1, st);
    } else {
      rc = run_conv(h, blk.c3, o2, n, h2, w2, r, dst, st);
    }
    if (rc) return rc;
    a = dst;
    cur = role[3];
    o1_ready = chain ? role[0] : -1;
    *hh = h2;
    *ww = w2;
  }
  *y = a;
  return 0;
}

// The BasicBlock walk (resnet.py:19-48) on x [n, hh, ww, 64]: conv1 (3x3 / stride, ReLU), then conv2 (3x3) + shortcut
// + ReLU in one launch -- the identity as the epilogue's residual, a downsample as the K-concatenated 1x1 of
// ctl_conv3x3_dual_nhwc_f16 (its stride-2 parity view needs even sides, which the stride-2 conv1 already requires).
// Three workspace slots of `slot` bytes: the block input (x_slot; < 0: a caller tensor that is never written), conv1's
// output and the block output.  The last block writes `out` when it is given.  *y = the trunk output [n, *hh, *ww, 512].
static int run_basic_blocks(ctl_trunk* h, const void* x, int x_slot, int n, int* hh, int* ww, char* ws, size_t slot,
                            void* out, const void** y, cudaStream_t st) {
  int rc;
  const void* a = x;
  int cur = x_slot;
  for (size_t bi = 0; bi < h->blocks.size(); ++bi) {
    const TrunkBlock& blk = h->blocks[bi];
    const int o1_slot = (cur + 1) % 3, dst_slot = (cur + 2) % 3;
    void* o1 = ws + o1_slot * slot;
    void* dst = out && bi + 1 == h->blocks.size() ? out : ws + dst_slot * slot;
    const int h1 = *hh, w1 = *ww, s = blk.c1.stride;
    const int h2 = (h1 + 2 - 3) / s + 1, w2 = (w1 + 2 - 3) / s + 1;
    if ((rc = run_conv(h, blk.c1, a, n, h1, w1, nullptr, o1, st))) return rc;
    if (blk.has_down) {
      ++h->launches;
      rc = ctl_conv3x3_dual_nhwc_f16(o1, blk.c2.cin, a, h1, w1, blk.down.cin, s, n, blk.dual_w, blk.dual_b, dst, blk.c2.cout,
                                     1, st);
    } else {
      rc = run_conv(h, blk.c2, o1, n, h2, w2, a, dst, st);
    }
    if (rc) return rc;
    a = dst;
    cur = dst_slot;
    *hh = h2;
    *ww = w2;
  }
  *y = a;
  return 0;
}

static int run_walk(ctl_trunk* h, const void* x, int x_slot, int n, int* hh, int* ww, char* ws, size_t slot, void* out,
                    const void** y, cudaStream_t st) {
  return h->block == CTL_BLOCK_BASIC ? run_basic_blocks(h, x, x_slot, n, hh, ww, ws, slot, out, y, st)
                                     : run_blocks(h, x, x_slot, n, hh, ww, ws, slot, out, y, st);
}

// global average pool (+ the folded BatchNorm1d head when out_emb is given)
static int run_head(ctl_trunk* h, const void* y, int n, int hw, float* out_feat, float* out_emb, cudaStream_t st) {
  ++h->launches;
  return ctl_gap_bn_nhwc_f16(y, n, hw, h->feature_dim, out_emb ? h->head_scale : nullptr, out_emb ? h->head_shift : nullptr, out_feat,
                             out_emb, st);
}

}  // namespace ctl

extern "C" {

size_t ctl_embed_workspace_bytes(const ctl_trunk* h, int32_t n, int32_t hgt, int32_t wid) {
  if (!h || n < 1 || hgt < 8 || wid < 8) return 0;
  const size_t slot = block_slot_bytes(h, n, pool_side(stem_side(hgt)), pool_side(stem_side(wid)));
  if (h->block == CTL_BLOCK_BASIC)  // the stem's temporary starts at slot 1 (ctl_embed_forward) and may span several
    return std::max(3 * slot, slot + stem_tmp_bytes(n, hgt, wid));
  return 5 * std::max(slot, stem_tmp_bytes(n, hgt, wid));
}

int ctl_embed_stem(ctl_trunk* h, const void* x, int32_t n, int32_t hgt, int32_t wid, const float* mean3_host,
                   const float* std3_host, void* out_nhwc, void* workspace, size_t workspace_bytes, ctl_stream_t stream) {
  CTL_CHECK_ARG(h && x && out_nhwc && workspace, "null pointer");
  CTL_CHECK_ARG(n >= 1 && hgt >= 8 && wid >= 8, "bad input shape");
  CTL_CHECK_ARG((mean3_host == nullptr) == (std3_host == nullptr), "uint8 input needs both mean3_host and std3_host");
  CTL_CHECK_ARG(!mean3_host || fused_stem_fits(hgt, wid), "uint8 input needs h %% 4 == 0 and an even w <= 128 (got %dx%d)", hgt,
                wid);
  int rc = check_workspace(ctl_embed_workspace_bytes(h, n, hgt, wid), workspace_bytes);
  if (rc || (rc = begin_call(h))) return rc;
  return run_stem(h, x, mean3_host, std3_host, n, hgt, wid, out_nhwc, workspace, (cudaStream_t)stream);
}

int ctl_embed_blocks(ctl_trunk* h, const void* x_nhwc, int32_t n, int32_t hgt, int32_t wid, void* out_nhwc, void* workspace,
                     size_t workspace_bytes, ctl_stream_t stream) {
  CTL_CHECK_ARG(h && x_nhwc && out_nhwc && workspace, "null pointer");
  CTL_CHECK_ARG(n >= 1 && hgt >= 2 && wid >= 2, "bad activation shape");
  const size_t slot = block_slot_bytes(h, n, hgt, wid);
  int rc = check_workspace(block_slots(h) * slot, workspace_bytes);
  if (rc || (rc = begin_call(h))) return rc;
  int hh = hgt, ww = wid;
  const void* y = nullptr;
  return run_walk(h, x_nhwc, -1, n, &hh, &ww, static_cast<char*>(workspace), slot, out_nhwc, &y, (cudaStream_t)stream);
}

int ctl_embed_head(ctl_trunk* h, const void* x_nhwc, int32_t n, int32_t hw, float* out_feat, float* out_emb,
                   ctl_stream_t stream) {
  CTL_CHECK_ARG(h && x_nhwc && (out_feat || out_emb), "null pointer");
  CTL_CHECK_ARG(n >= 1 && hw >= 1, "bad activation shape");
  CTL_CHECK_ARG(out_emb == nullptr || h->has_head, "out_emb needs the bn_head.* tensors in ctl_weights_pack");
  int rc = begin_call(h);
  if (rc) return rc;
  return run_head(h, x_nhwc, n, hw, out_feat, out_emb, (cudaStream_t)stream);
}

int ctl_embed_forward(ctl_trunk* h, const float* x_nchw, int32_t n, int32_t hgt, int32_t wid, float* out_feat, float* out_emb,
                      void* workspace, size_t workspace_bytes, ctl_stream_t stream) {
  CTL_CHECK_ARG(h && x_nchw && workspace && (out_feat || out_emb), "null pointer");
  CTL_CHECK_ARG(n >= 1 && hgt >= 8 && wid >= 8, "bad input shape");
  CTL_CHECK_ARG(out_emb == nullptr || h->has_head, "out_emb needs the bn_head.* tensors in ctl_weights_pack");
  int rc = check_workspace(ctl_embed_workspace_bytes(h, n, hgt, wid), workspace_bytes);
  if (rc || (rc = begin_call(h))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int hh = pool_side(stem_side(hgt)), ww = pool_side(stem_side(wid));
  const size_t slot = block_slot_bytes(h, n, hh, ww);
  char* ws = static_cast<char*>(workspace);
  // the stem writes slot 0; the tensor-core stem's temporary (at most one activation) starts at slot 1
  if ((rc = run_stem(h, x_nchw, nullptr, nullptr, n, hgt, wid, ws, ws + slot, st))) return rc;
  const void* y = nullptr;
  if ((rc = run_walk(h, ws, 0, n, &hh, &ww, ws, slot, nullptr, &y, st))) return rc;
  return run_head(h, y, n, hh * ww, out_feat, out_emb, st);
}

int32_t ctl_embed_launches(const ctl_trunk* h) { return h ? h->launches : 0; }

}  // extern "C"
