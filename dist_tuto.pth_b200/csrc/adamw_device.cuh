// The AdamW update of one element, shared by adamw_flat_kernel (adamw.cu) and the AdamW instance of the sharded optimizer
// kernel (sharded_sgd.cu), so that both compute the same bits.
//
// torch.optim.AdamW (amsgrad=False, maximize=False, single-tensor order), update t = steps + 1:
//   p   = p * (1 - lr*wd)                                   __fmul_rn  (decay == 1 without weight decay: exact)
//   d   = g - m;  m = w1 < 0.5 ? fmaf(w1, d, m)             lerp(m, g, w1) with w1 = 1 - beta1, in ATen's two branches
//                                 : fmaf(-d, 1 - w1, g)
//   v   = fmaf((1 - beta2) * g, g, v * beta2)               mul_(beta2).addcmul_(g, g, value=1 - beta2)
//   den = sqrt(v) / sqrt(1 - beta2^t) + eps                 __fsqrt_rn, __fdiv_rn, __fadd_rn
//   p   = fmaf(-(lr / (1 - beta1^t)), m / den, p)           addcdiv_(m, den, value=-step_size), m / den by __fdiv_rn
// The host computes 1 - lr*wd, lr / bc1 and sqrt(bc2) in fp64 per update, as torch's non-capturable path does, and rounds
// each once to fp32.  The build uses --use_fast_math, so every rounding that matters is spelled out: no contraction or
// approximate sqrt / division can change these bits.  tests/adamw_model.py is the same sequence on the CPU.
#pragma once
#include "adamw.h"
#include "common.cuh"

namespace b2 {

// The moment lines of the sequence above, shared with LAMB (layerwise_device.cuh).  S: any type with the fields w1 (1 - beta1),
// beta2 and c2 (1 - beta2): AdamwScalars or LwArgs.
template <class S>
__device__ __forceinline__ void adam_moments(float& m, float& v, float g, const S& s) {
  const float d = __fsub_rn(g, m);
  m = s.w1 < 0.5f ? fmaf(s.w1, d, m) : fmaf(-d, __fsub_rn(1.f, s.w1), g);
  v = fmaf(__fmul_rn(s.c2, g), g, __fmul_rn(v, s.beta2));
}

__device__ __forceinline__ void adamw_elem(float& p, float& m, float& v, float g, const AdamwScalars& s) {
  p = __fmul_rn(p, s.decay);
  adam_moments(m, v, g, s);
  const float den = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), s.sbc2), s.eps);
  p = fmaf(-s.step_size, __fdiv_rn(m, den), p);
}

__device__ __forceinline__ void adamw4(float4& p, float4& m, float4& v, float4 g, const AdamwScalars& s) {
  adamw_elem(p.x, m.x, v.x, g.x, s);
  adamw_elem(p.y, m.y, v.y, g.y, s);
  adamw_elem(p.z, m.z, v.z, g.z, s);
  adamw_elem(p.w, m.w, v.w, g.w, s);
}

}  // namespace b2
