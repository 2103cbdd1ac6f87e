// b200ot — the kernel kinds of the convolutions and the coordinates each one is evaluated in, for both paths
// (b200ot_kernel_conv.cu: CUDA cores, b200ot_tc.cu: tensor cores).
#pragma once
#include "common.cuh"
#include "host_util.cuh"

namespace b200ot {

struct ConvScales {
  float scale;   // coordinate scale
  float clampq;  // clamp on the scaled squared distance
  int direct;
  int extra;
};

// `kind` may carry B200OT_KERNEL_UNCLAMPED (laplacian / energy with pykeops' unclamped sqrt)
inline int kind_base(int kind) { return kind & 0xff; }
inline bool valid_kind(int kind) {
  return kind_base(kind) >= 0 && kind_base(kind) <= 2 && (kind & ~(0xff | B200OT_KERNEL_UNCLAMPED)) == 0;
}

// blur is the length scale of the gaussian and laplacian kernels; the energy kernel has none
inline bool blur_ok(int kind, float blur) { return kind_base(kind) == B200OT_KERNEL_ENERGY || blur > 0.f; }

inline ConvScales conv_scales(int kind_flags, float blur) {
  ConvScales c;
  const int kind = kind_base(kind_flags);
  const float clamp = cost_clamp(kind_flags);  // B200OT_KERNEL_UNCLAMPED == B200OT_P_UNCLAMPED
  if (kind == B200OT_KERNEL_GAUSSIAN) {
    c.scale = sqrtf(kLog2e) / blur;  // 2^(-|X-Y|^2/2) = exp(-|x-y|^2 / (2 blur^2))
    c.clampq = 0.f;
    c.direct = 0;
    c.extra = 2;
  } else if (kind == B200OT_KERNEL_LAPLACIAN) {
    c.scale = kLog2e / blur;  // 2^(-|X-Y|) = exp(-|x-y| / blur)
    c.clampq = kLog2e * kLog2e * clamp;
    c.direct = 1;
    c.extra = 1;
  } else {
    c.scale = 1.f;
    c.clampq = clamp;
    c.direct = 1;
    c.extra = 1;
  }
  return c;
}

}  // namespace b200ot
