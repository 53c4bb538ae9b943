// The ResNet both trunk handles are built from (ctl_trunk in trunk.cu, ctl_trainer in trunk_train.cu): which blocks
// exist, each convolution's state_dict names and shape, where the downsamples are and which bn1 is IBN-a --
// ResNet (modelling/backbones/resnet.py:19-120) and ResNet_IBN (resnet_ibn_a.py:34-124).  Also the plumbing the two
// handles share: named-tensor lookup, handle-owned allocations, the stem's operand pack.  Host only.
#pragma once
#include <cuda_fp16.h>

#include <array>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.h"

namespace ctl {

static constexpr float BN_EPS = 1e-5f;  // every BatchNorm / InstanceNorm of the trunk and the BatchNorm1d head

inline int stem_side(int s) { return (s + 6 - 7) / 2 + 1; }  // conv1 7x7 / 2, pad 3
inline int pool_side(int s) { return (s + 2 - 3) / 2 + 1; }  // maxpool 3x3 / 2, pad 1

// One convolution and the normalisation after it.  in_half > 0 (IBN-a bn1, resnet_ibn_a.py:18-32): InstanceNorm on
// channels [0, in_half), BatchNorm on [in_half, cout), so ReLU in a conv epilogue starts at channel in_half.
struct ConvLayout {
  std::string conv;  // "<conv>.weight" [cout][cin][k][k]
  std::string bn;    // "<bn>.weight|bias|running_mean|running_var" [cout - in_half]
  std::string in;    // "<in>.weight|bias" [in_half]; empty without IBN
  int cin = 0, cout = 0, k = 1, stride = 1, relu = 1, in_half = 0;
};

// A block whose convolutions are `Conv`s: a ConvLayout plus what a handle keeps per convolution.  A BasicBlock has no
// c3: c1 and c2 are its two 3x3 convolutions.
template <class Conv>
struct BlockLayout {
  std::string prefix;  // "layer<stage>.<block>"
  Conv c1, c2, c3, down;
  bool bottleneck = true, has_down = false;
  // state_dict order: conv1, conv2, [conv3], [downsample]; nullptr where a block has no such convolution
  std::array<Conv*, 4> state_dict_order() {
    return {&c1, &c2, bottleneck ? &c3 : nullptr, has_down ? &down : nullptr};
  }
  // forward order: conv1, conv2, [downsample], conv3 of a bottleneck; conv1, [downsample], conv2 of a BasicBlock (its
  // conv2 adds the shortcut, so the downsample runs first)
  std::array<const Conv*, 4> forward_order() const {
    return {&c1, bottleneck ? &c2 : nullptr, has_down ? &down : nullptr, bottleneck ? &c3 : &c2};
  }
};

// Checks the arguments of a trunk handle's create call and lays out ResNet(block, stage_blocks): *feature_dim = 2048
// (bottleneck) or 512 (BasicBlock), *blocks = every block in forward order.  `Block` derives from BlockLayout<Conv>.
template <class Block>
int resnet_layout(int32_t block, int32_t ibn, int32_t last_stride, const int32_t stage_blocks[4], int* feature_dim,
                  std::vector<Block>* blocks) {
  CTL_CHECK_ARG(stage_blocks != nullptr, "null pointer");
  CTL_CHECK_ARG(block == CTL_BLOCK_BOTTLENECK || block == CTL_BLOCK_BASIC,
                "block = %d: expected CTL_BLOCK_BOTTLENECK (0) or CTL_BLOCK_BASIC (1)", block);
  CTL_CHECK_ARG(block == CTL_BLOCK_BOTTLENECK || !ibn, "IBN-a is defined for bottleneck blocks only (resnet_ibn_a.py)");
  CTL_CHECK_ARG(last_stride == 1 || last_stride == 2, "last_stride must be 1 or 2 (config/defaults.py:24)");
  for (int li = 0; li < 4; ++li)
    CTL_CHECK_ARG(stage_blocks[li] >= 1, "stage_blocks[%d] = %d: every stage needs at least one block", li, stage_blocks[li]);
  const bool bottleneck = block == CTL_BLOCK_BOTTLENECK;
  const int expansion = bottleneck ? 4 : 1;
  *feature_dim = 512 * expansion;
  blocks->clear();
  int inplanes = 64;
  for (int li = 0; li < 4; ++li) {
    const int planes = 64 << li, out = planes * expansion;
    for (int bi = 0; bi < stage_blocks[li]; ++bi) {
      Block b;
      const std::string p = "layer" + std::to_string(li + 1) + "." + std::to_string(bi);
      auto set = [&p](ConvLayout& c, const char* conv, const char* bn, int cin, int cout, int k, int stride) {
        c = ConvLayout{p + conv, p + bn, "", cin, cout, k, stride};
      };
      // resnet.py:19-87,94-112: the first block of layers 2-4 has stride 2 (layer4: last_stride) in conv1 of a
      // BasicBlock, in the 3x3 conv2 of a bottleneck, and in the downsample, which exists where the stride or the
      // width changes
      const int stride = bi == 0 && li > 0 ? (li == 3 ? last_stride : 2) : 1;
      b.prefix = p;
      b.bottleneck = bottleneck;
      if (bottleneck) {
        set(b.c1, ".conv1", ".bn1", inplanes, planes, 1, 1);
        set(b.c2, ".conv2", ".bn2", planes, planes, 3, stride);
        set(b.c3, ".conv3", ".bn3", planes, out, 1, 1);
        if (ibn && planes != 512) {  // resnet_ibn_a.py:116-119
          b.c1.bn = p + ".bn1.BN";
          b.c1.in = p + ".bn1.IN";
          b.c1.in_half = planes / 2;
        }
      } else {
        set(b.c1, ".conv1", ".bn1", inplanes, planes, 3, stride);
        set(b.c2, ".conv2", ".bn2", planes, planes, 3, 1);
      }
      b.has_down = stride != 1 || inplanes != out;
      if (b.has_down) {
        set(b.down, ".downsample.0", ".downsample.1", inplanes, out, 1, stride);
        b.down.relu = 0;
      }
      inplanes = out;
      blocks->push_back(b);
    }
  }
  return 0;
}

// name -> device tensor of one call's ctl_named_tensor / ctl_named_buffer list; `call` is the entry point errors name
struct NamedMap {
  struct Ref {
    float* data;
    long long numel;
  };
  const char* call = "";
  std::unordered_map<std::string, Ref> refs;
};

// Indexes the `n` entries of `list` (`what` names them in errors); an entry without a name is CTL_ERR_INVALID_ARGUMENT.
template <class Named>
int index_named(const Named* list, int32_t n, const char* call, const char* what, NamedMap* out) {
  out->call = call;
  for (int i = 0; i < n; ++i) {
    CTL_CHECK_ARG(list[i].name != nullptr, "%s %d has no name", what, i);
    out->refs[list[i].name] = NamedMap::Ref{const_cast<float*>(list[i].data), (long long)list[i].numel};
  }
  return 0;
}

// The tensor `name` of `numel` elements, or nullptr.  A mis-sized tensor, or a missing one when `required`, sets *rc to
// CTL_ERR_INVALID_ARGUMENT and an error naming the entry point, the tensor's role `what` and the tensor.
inline float* lookup(const NamedMap& m, const std::string& name, long long numel, int* rc, const char* what = "tensor",
                     bool required = true) {
  auto it = m.refs.find(name);
  if (it == m.refs.end() || it->second.data == nullptr) {
    if (required) {
      set_error("%s: %s '%s' is missing", m.call, what, name.c_str());
      *rc = CTL_ERR_INVALID_ARGUMENT;
    }
    return nullptr;
  }
  if (it->second.numel != numel) {
    set_error("%s: %s '%s' has %lld elements, expected %lld", m.call, what, name.c_str(), it->second.numel, numel);
    *rc = CTL_ERR_INVALID_ARGUMENT;
    return nullptr;
  }
  return it->second.data;
}

// cudaMalloc of `count` Ts that handle `h` frees in its destroy call; nullptr when out of memory
template <typename T, class Handle>
T* dev_alloc(Handle* h, size_t count) {
  void* p = nullptr;
  if (cudaMalloc(&p, count * sizeof(T)) != cudaSuccess) return nullptr;
  h->owned.push_back(p);
  return static_cast<T*>(p);
}

// trunk.cu: conv1.weight [64][3][7][7] -> the tensor-core stem's operand w192 [64][192] (ctl_stem_conv7x7_tc) and, when
// w3 is given, the fused stem's w3 [28][64][8] (ctl_stem_pool_fused), with bn1 folded in and its bias written -- or,
// with gamma == nullptr, unfolded: scale 1, and w * 1 == w exactly.
int stem_pack(const float* w, const float* gamma, const float* beta, const float* mean, const float* var, __half* w192,
              __half* w3, float* bias, cudaStream_t st);

}  // namespace ctl
