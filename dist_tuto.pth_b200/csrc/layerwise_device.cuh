// The per-element pieces of FlatLAMB and FlatLARS (layerwise.cu).  The build uses --use_fast_math, so every rounding is
// spelled out; tests/layerwise_model.py is the same sequence on the CPU.
//
// LAMB, update t:  m, v as AdamW (adam_moments);  den = sqrt(v) / sqrt(1 - beta2^t) + eps
//                  u = fmaf(wd_l, p, (m / den) * (1 / (1 - beta1^t)));   p = fmaf(-(lr * r), u, p)
// LARS:            d = r * fmaf(wd_l, p, g);  m = fmaf(mu, m, d);  p = fmaf(-lr, nesterov ? fmaf(mu, m, d) : m, p)
// wd_l is weight_decay for a tensor with a trust ratio and 0 for an excluded one; r is the tensor's trust ratio.
#pragma once
#include "adamw_device.cuh"
#include "layerwise.h"

namespace b2 {

__device__ __forceinline__ float lamb_u(float p, float m, float v, float wd, const LwArgs& a) {
  const float den = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), a.sbc2), a.eps);
  return fmaf(wd, p, __fmul_rn(__fdiv_rn(m, den), a.rbc1));
}

__device__ __forceinline__ void lars_elem(float& p, float& m, float g, float r, float wd, const LwArgs& a) {
  const float d = __fmul_rn(r, fmaf(wd, p, g));
  m = fmaf(a.mu, m, d);
  p = fmaf(-a.lr, a.nesterov ? fmaf(a.mu, m, d) : m, p);
}

}  // namespace b2
