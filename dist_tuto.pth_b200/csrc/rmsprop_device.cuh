// The RMSprop update of one element, shared by rmsprop_flat_kernel (rmsprop.cu) and the RMSprop instances of the sharded
// optimizer kernel (sharded_sgd.cu), so that all of them compute the same bits.
//
// torch.optim.RMSprop (maximize=False, single-tensor order), with the fused multiply-adds where torch's CUDA kernels contract:
//   g   = fmaf(wd, p, g)                                        grad.add(param, alpha=wd), only when wd != 0
//   sq  = fmaf(c * g, g, sq * alpha)                            square_avg.mul_(alpha).addcmul_(g, g, value=1 - alpha)
//   centered:
//     d   = g - ga;  ga = |c| < 0.5 ? fmaf(c, d, ga)            grad_avg.lerp_(g, 1 - alpha), ATen's two branches
//                               : fmaf(-d, 1 - c, g)
//     avg = sqrt(fmaf(-ga, ga, sq)) + eps                       square_avg.addcmul(ga, ga, value=-1).sqrt_().add_(eps)
//   else:
//     avg = sqrt(sq) + eps                                      square_avg.sqrt().add_(eps)
//   momentum:
//     buf = buf * mu + g / avg                                  buf.mul_(momentum).addcdiv_(g, avg)
//     p   = fmaf(-lr, buf, p)                                   param.add_(buf, alpha=-lr)
//   else:
//     p   = fmaf(-lr, g / avg, p)                               param.addcdiv_(g, avg, value=-lr)
// with c = 1 - alpha computed in fp64 by the host and every scalar rounded once to fp32.  The build uses --use_fast_math,
// so every rounding is spelled out (__fmul_rn, __fadd_rn, __fdiv_rn, __fsqrt_rn, fmaf): no contraction or approximate
// square root / division can change these bits.  `centered` and `momentum` are uniform per launch; an absent state is never
// read or written.  tests/rmsprop_model.py is the same sequence on the CPU.
#pragma once
#include "common.cuh"
#include "rmsprop.h"

namespace b2 {

__device__ __forceinline__ void rmsprop_elem(float& p, float& sq, float& ga, float& buf, float g, const RmspropScalars& s) {
  if (s.wd != 0.f) g = fmaf(s.wd, p, g);
  sq = fmaf(__fmul_rn(s.c, g), g, __fmul_rn(sq, s.alpha));
  float avg;
  if (s.centered) {
    const float d = __fsub_rn(g, ga);
    ga = fabsf(s.c) < 0.5f ? fmaf(s.c, d, ga) : fmaf(-d, __fsub_rn(1.f, s.c), g);
    avg = __fsqrt_rn(fmaf(-ga, ga, sq));
  } else {
    avg = __fsqrt_rn(sq);
  }
  avg = __fadd_rn(avg, s.eps);
  if (s.momentum) {
    buf = __fadd_rn(__fmul_rn(buf, s.mu), __fdiv_rn(g, avg));
    p = fmaf(-s.lr, buf, p);
  } else {
    p = fmaf(-s.lr, __fdiv_rn(g, avg), p);
  }
}

__device__ __forceinline__ void rmsprop4(float4& p, float4& sq, float4& ga, float4& buf, float4 g, const RmspropScalars& s) {
  rmsprop_elem(p.x, sq.x, ga.x, buf.x, g.x, s);
  rmsprop_elem(p.y, sq.y, ga.y, buf.y, g.y, s);
  rmsprop_elem(p.z, sq.z, ga.z, buf.z, g.z, s);
  rmsprop_elem(p.w, sq.w, ga.w, buf.w, g.w, s);
}

}  // namespace b2
