// Capturable FlatSGD / FlatAdamW (ops/optim.py, capturable=True): the scalars of an update live on the device, so a captured
// CUDA graph replays the lr schedule and AdamW's bias corrections instead of freezing the values of the capture.
//
// Device state of one optimizer: a uint64 step counter (updates applied so far), the fp64 hyper-parameter table FlatHyper and
// the scalar block FlatScalars (flat_scalars.h).  flat_scalars_kernel (flat_scalars.cu), one CTA, adds 1 to the counter and
// fills the block for the next update; with advance = 0 it only fills the block (at construction, after load_state_dict and
// after the host uploads new group values).  For the update run when the counter reads s, with t = s + 1:
//   lr_t       = lr_schedule_lr(sched, fp32(lr_g), s)                      lr_schedule.h, unchanged
//   wd         = fp32(wd_g)
//   beta^t     = exponentiation by squaring with __dmul_rn (flat_pow)      stateless in t: a resumed run gets the same bits
//   decay      = fp32(1 - lr_t*wd_g)                                       wd_g in fp64, as the host computes it
//   step_size  = fp32(__ddiv_rn(lr_t, 1 - beta1^t))
//   sbc2       = fp32(__dsqrt_rn(1 - beta2^t))
//   w1, beta2, c2, eps = fp32(1 - beta1), fp32(beta2), fp32(1 - beta2), fp32(eps)
// Every value is rounded once to fp32.
//
// Contract:
//   * given the same scalars, a capturable instance computes bit for bit what its existing instance computes: it loads the
//     block once per CTA through shared memory and then runs the unchanged per-element code (sgd4, adamw_elem, clip_coef);
//   * the block is bit for bit the CPU model tests/capturable_model.py (the same squaring order, explicitly rounded fp64);
//   * it agrees with the host's adamw_scalars within one fp32 ulp: Python's b ** t is not repeated squaring, and ** 0.5 is
//     not sqrt, so the last fp64 bits may differ;
//   * the cosine schedule keeps lr_schedule.h's documented one ulp against LRSchedule.lr_at.
#pragma once
#include "flat_scalars.h"
#include "sgd_device.cuh"

namespace b2 {

// b^t by squaring, the factors taken from the lowest bit of t up; every product rounded to nearest (no contraction)
__device__ __forceinline__ double flat_pow(double b, unsigned long long t) {
  double r = 1.0;
  while (t != 0ull) {
    if (t & 1ull) r = __dmul_rn(r, b);
    b = __dmul_rn(b, b);
    t >>= 1;
  }
  return r;
}

// Cooperative copy of the block's field `src` (global) to `dst` (shared), one 32-bit word per thread and pass; the caller
// synchronises the CTA before reading it.
template <class T>
__device__ __forceinline__ void flat_block_load(T& dst, const T& src) {
  static_assert(sizeof(T) % 4 == 0, "the block's fields are fp32 words");
  const uint32_t* s = reinterpret_cast<const uint32_t*>(&src);
  uint32_t* d = reinterpret_cast<uint32_t*>(&dst);
  for (int i = threadIdx.x; i < (int)(sizeof(T) / 4); i += blockDim.x) d[i] = __ldg(s + i);
}

// The clip coefficient of the capturable unsharded instances, as their existing instances take it: the norm
// sqrt(sum of sqnorms[0, n_buckets)) in fp64, rounded once, then clip_coef; CTA 0 also stores the norm.  Thread 0 only.
__device__ __forceinline__ float flat_clip_coef(const double* __restrict__ sqnorms, int n_buckets, float max_norm,
                                                float* grad_norm_out) {
  double q = 0.0;
  for (int k = 0; k < n_buckets; ++k) q += sqnorms[k];
  const float nrm = __double2float_rn(__dsqrt_rn(q));
  if (blockIdx.x == 0 && grad_norm_out != nullptr) *grad_norm_out = nrm;
  return clip_coef(nrm, max_norm);
}

}  // namespace b2
