// FlatAdamW's update of one gradient bucket on sm_90a (ops/optim.py): AdamW over the flat fp32 parameters, first and second
// moments and averaged gradients, one launch per bucket, streaming the four arrays once and re-zeroing the gradients in the
// same pass.  The per-element sequence is adamw_elem (adamw_device.cuh).
#include "adamw_device.cuh"
#include "param_groups.cuh"
#include "sgd_device.cuh"
#include "flat_scalars.cuh"

namespace b2 {

// kClip: g *= coef first, coef = clip_coef(total norm) with the norm sqrt(sum of sqnorms[0, n_buckets)) taken in fp64 and
// rounded once (grad_sqnorm_kernel fills sqnorms), as sgd_flat_clip_kernel does.  The kClip = false instance has no clip code.
// kScaled: the gradient is g * amp_inv_scale(grad_scale) (sgd_device.cuh), unscaled before the clip coefficient.
template <bool kClip, bool kScaled>
__global__ void __launch_bounds__(256) adamw_flat_kernel(float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                                                         float* __restrict__ g, size_t n, AdamwScalars s, int zero_grad,
                                                         const double* __restrict__ sqnorms, int n_buckets, float max_norm,
                                                         float* grad_norm_out, const float* grad_scale) {
  float c = 1.f;
  if constexpr (kClip) {
    __shared__ float s_coef;
    if (threadIdx.x == 0) {
      double q = 0.0;
      for (int k = 0; k < n_buckets; ++k) q += sqnorms[k];
      const float nrm = __double2float_rn(__dsqrt_rn(q));
      s_coef = clip_coef(nrm, max_norm);
      if (blockIdx.x == 0 && grad_norm_out != nullptr) *grad_norm_out = nrm;
    }
    __syncthreads();
    c = s_coef;
  }
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n4 = n / 4;
  const float inv = kScaled ? amp_inv_scale(grad_scale) : 1.f;
  if (i < n4) {
    float4 gv = reinterpret_cast<const float4*>(g)[i];
    float4 pv = reinterpret_cast<float4*>(p)[i];
    float4 mv = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    if constexpr (kScaled) gv = amp_unscale4(gv, inv);
    if constexpr (kClip) {
      gv.x = __fmul_rn(gv.x, c); gv.y = __fmul_rn(gv.y, c); gv.z = __fmul_rn(gv.z, c); gv.w = __fmul_rn(gv.w, c);
    }
    adamw4(pv, mv, vv, gv, s);
    reinterpret_cast<float4*>(p)[i] = pv;
    reinterpret_cast<float4*>(m)[i] = mv;
    reinterpret_cast<float4*>(v)[i] = vv;
    if (zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (i < n - n4 * 4) {                        // tail (< 4 elements): threads 0..2 of CTA 0, one element each
    const size_t t = n4 * 4 + i;
    const float gl = kScaled ? amp_unscale(g[t], inv) : g[t];
    const float gt = kClip ? __fmul_rn(gl, c) : gl;
    adamw_elem(p[t], m[t], v[t], gt, s);
    if (zero_grad) g[t] = 0.f;
  }
}

// adamw_flat_kernel with parameter groups: parameter vector i takes decay and step_size of group map[i] (param_groups.cuh),
// the other five scalars are shared; the tail (< 4 elements) shares the map entry of its vector.
template <bool kClip, bool kScaled>
__global__ void __launch_bounds__(256) adamw_flat_grouped_kernel(float* __restrict__ p, float* __restrict__ m,
                                                                 float* __restrict__ v, float* __restrict__ g, size_t n,
                                                                 const uint8_t* __restrict__ map, AdamwScalars s, AdamwGroups gs,
                                                                 int zero_grad, const double* __restrict__ sqnorms, int n_buckets,
                                                                 float max_norm, float* grad_norm_out, const float* grad_scale) {
  float c = 1.f;
  if constexpr (kClip) {
    __shared__ float s_coef;
    if (threadIdx.x == 0) {
      double q = 0.0;
      for (int k = 0; k < n_buckets; ++k) q += sqnorms[k];
      const float nrm = __double2float_rn(__dsqrt_rn(q));
      s_coef = clip_coef(nrm, max_norm);
      if (blockIdx.x == 0 && grad_norm_out != nullptr) *grad_norm_out = nrm;
    }
    __syncthreads();
    c = s_coef;
  }
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n4 = n / 4;
  const float inv = kScaled ? amp_inv_scale(grad_scale) : 1.f;
  if (i < n4) {
    const int gid = map[i];
    AdamwScalars sg = s;
    sg.decay = gs.decay[gid];
    sg.step_size = gs.step_size[gid];
    float4 gv = reinterpret_cast<const float4*>(g)[i];
    float4 pv = reinterpret_cast<float4*>(p)[i];
    float4 mv = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    if constexpr (kScaled) gv = amp_unscale4(gv, inv);
    if constexpr (kClip) {
      gv.x = __fmul_rn(gv.x, c); gv.y = __fmul_rn(gv.y, c); gv.z = __fmul_rn(gv.z, c); gv.w = __fmul_rn(gv.w, c);
    }
    adamw4(pv, mv, vv, gv, sg);
    reinterpret_cast<float4*>(p)[i] = pv;
    reinterpret_cast<float4*>(m)[i] = mv;
    reinterpret_cast<float4*>(v)[i] = vv;
    if (zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (i < n - n4 * 4) {                        // tail (< 4 elements): threads 0..2 of CTA 0, one element each
    const size_t t = n4 * 4 + i;
    const int gid = map[n4];
    AdamwScalars sg = s;
    sg.decay = gs.decay[gid];
    sg.step_size = gs.step_size[gid];
    const float gl = kScaled ? amp_unscale(g[t], inv) : g[t];
    const float gt = kClip ? __fmul_rn(gl, c) : gl;
    adamw_elem(p[t], m[t], v[t], gt, sg);
    if (zero_grad) g[t] = 0.f;
  }
}

// Capturable instances of adamw_flat_kernel and adamw_flat_grouped_kernel (flat_scalars.cuh): the AdamwScalars (kGrouped:
// also every group's decay and step_size) come from the scalar block `blk`, loaded once per CTA through shared memory.  The
// per-element sequence is adamw_elem, so the same scalars give the same bits.  kScaled: GradScaler's step, as in
// sgd_flat_cap_kernel (found_inf != 0: only the zeroing; grad_scale null: already unscaled).
template <bool kClip, bool kGrouped, bool kScaled>
__global__ void __launch_bounds__(256) adamw_flat_cap_kernel(float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                                                             float* __restrict__ g, size_t n, const uint8_t* __restrict__ map,
                                                             const FlatScalars* __restrict__ blk, int zero_grad,
                                                             const double* __restrict__ sqnorms, int n_buckets, float max_norm,
                                                             float* grad_norm_out, const float* grad_scale, const float* found_inf) {
  __shared__ float s_coef;
  __shared__ AdamwScalars s_s;
  __shared__ AdamwGroups s_gs;
  if constexpr (kScaled) {
    if (__ldg(found_inf) != 0.f) {
      amp_skip_zero(g, n, zero_grad);
      return;
    }
  }
  flat_block_load(s_s, blk->adamw);
  if constexpr (kGrouped) flat_block_load(s_gs, blk->adamw_groups);
  if constexpr (kClip) {
    if (threadIdx.x == 0) s_coef = flat_clip_coef(sqnorms, n_buckets, max_norm, grad_norm_out);
  }
  __syncthreads();
  const float c = kClip ? s_coef : 1.f;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n4 = n / 4;
  const float inv = kScaled && grad_scale != nullptr ? amp_inv_scale(grad_scale) : 1.f;
  if (i < n4) {
    AdamwScalars sg = s_s;
    if constexpr (kGrouped) {
      const int gid = map[i];
      sg.decay = s_gs.decay[gid];
      sg.step_size = s_gs.step_size[gid];
    }
    float4 gv = reinterpret_cast<const float4*>(g)[i];
    float4 pv = reinterpret_cast<float4*>(p)[i];
    float4 mv = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    if constexpr (kScaled) gv = amp_unscale4(gv, inv);
    if constexpr (kClip) {
      gv.x = __fmul_rn(gv.x, c); gv.y = __fmul_rn(gv.y, c); gv.z = __fmul_rn(gv.z, c); gv.w = __fmul_rn(gv.w, c);
    }
    adamw4(pv, mv, vv, gv, sg);
    reinterpret_cast<float4*>(p)[i] = pv;
    reinterpret_cast<float4*>(m)[i] = mv;
    reinterpret_cast<float4*>(v)[i] = vv;
    if (zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (i < n - n4 * 4) {                        // tail (< 4 elements): threads 0..2 of CTA 0, one element each
    const size_t t = n4 * 4 + i;
    AdamwScalars sg = s_s;
    if constexpr (kGrouped) {
      const int gid = map[n4];
      sg.decay = s_gs.decay[gid];
      sg.step_size = s_gs.step_size[gid];
    }
    const float gl = kScaled ? amp_unscale(g[t], inv) : g[t];
    const float gt = kClip ? __fmul_rn(gl, c) : gl;
    adamw_elem(p[t], m[t], v[t], gt, sg);
    if (zero_grad) g[t] = 0.f;
  }
}

}  // namespace b2

extern "C" {

// The capturable adamw_flat / adamw_flat_grouped (flat_scalars.cuh): the scalars come from the block `blk` on the device.
// `map`: null without groups, else one group id per parameter vector.  cudaErrorInvalidValue, without a launch, for a null
// pointer or clipping without sqnorms.
// found_inf / grad_scale: GradScaler's step, as in b2_sgd_flat_cap_launch.
int b2_adamw_flat_cap_launch(float* p, float* m, float* v, float* g, size_t n, const uint8_t* map, const b2::FlatScalars* blk,
                             int zero_grad, float max_norm, const double* sqnorms, int n_buckets, float* grad_norm_out,
                             const float* grad_scale, const float* found_inf, cudaStream_t stream) {
  if (p == nullptr || m == nullptr || v == nullptr || g == nullptr || blk == nullptr) return (int)cudaErrorInvalidValue;
  if (found_inf == nullptr && grad_scale != nullptr) return (int)cudaErrorInvalidValue;
  const bool clip = max_norm > 0.f;
  if (clip && (sqnorms == nullptr || n_buckets < 1 || !(max_norm < INFINITY))) return (int)cudaErrorInvalidValue;
  const size_t n4 = (n / 4) > 0 ? n / 4 : 1;
  const unsigned blocks = (unsigned)((n4 + 255) / 256);
  using namespace b2;
#define B2_ADAMW_CAP(C, G, S) adamw_flat_cap_kernel<C, G, S><<<blocks, 256, 0, stream>>>(p, m, v, g, n, map, blk, zero_grad, \
      C ? sqnorms : nullptr, C ? n_buckets : 0, C ? max_norm : 0.f, C ? grad_norm_out : nullptr, grad_scale, found_inf)
  const int k = (found_inf != nullptr ? 4 : 0) | (clip ? 2 : 0) | (map != nullptr ? 1 : 0);
  switch (k) {
    case 0: B2_ADAMW_CAP(false, false, false); break;
    case 1: B2_ADAMW_CAP(false, true, false); break;
    case 2: B2_ADAMW_CAP(true, false, false); break;
    case 3: B2_ADAMW_CAP(true, true, false); break;
    case 4: B2_ADAMW_CAP(false, false, true); break;
    case 5: B2_ADAMW_CAP(false, true, true); break;
    case 6: B2_ADAMW_CAP(true, false, true); break;
    default: B2_ADAMW_CAP(true, true, true); break;
  }
#undef B2_ADAMW_CAP
  return (int)cudaGetLastError();
}

// One AdamW update of a flat bucket of n elements on `stream`.  max_norm > 0: clipped by the norm of grad_sqnorm's n_buckets
// sums.  cudaErrorInvalidValue, without a launch, for a null pointer or clipping without sqnorms.
// grad_scale (fp32 on the device, or null): GradScaler's loss scale, unscaled by the kScaled instances.
int b2_adamw_flat_launch(float* p, float* m, float* v, float* g, size_t n, const b2::AdamwScalars* s, int zero_grad,
                         float max_norm, const double* sqnorms, int n_buckets, float* grad_norm_out, const float* grad_scale,
                         cudaStream_t stream) {
  if (p == nullptr || m == nullptr || v == nullptr || g == nullptr || s == nullptr) return (int)cudaErrorInvalidValue;
  const size_t n4 = (n / 4) > 0 ? n / 4 : 1;
  const unsigned blocks = (unsigned)((n4 + 255) / 256);
  using namespace b2;
  const bool scaled = grad_scale != nullptr;
  if (max_norm > 0.f) {
    if (sqnorms == nullptr || n_buckets < 1 || !(max_norm < INFINITY)) return (int)cudaErrorInvalidValue;
    if (scaled)
      adamw_flat_kernel<true, true><<<blocks, 256, 0, stream>>>(p, m, v, g, n, *s, zero_grad, sqnorms, n_buckets, max_norm,
                                                                grad_norm_out, grad_scale);
    else
      adamw_flat_kernel<true, false><<<blocks, 256, 0, stream>>>(p, m, v, g, n, *s, zero_grad, sqnorms, n_buckets, max_norm,
                                                                 grad_norm_out, nullptr);
  } else if (scaled) {
    adamw_flat_kernel<false, true><<<blocks, 256, 0, stream>>>(p, m, v, g, n, *s, zero_grad, nullptr, 0, 0.f, nullptr, grad_scale);
  } else {
    adamw_flat_kernel<false, false><<<blocks, 256, 0, stream>>>(p, m, v, g, n, *s, zero_grad, nullptr, 0, 0.f, nullptr, nullptr);
  }
  return (int)cudaGetLastError();
}

// The same update with parameter groups: `map` holds one group id per parameter vector (ceil(n / 4) ids), `gs` the per-group
// scalars of n_groups groups.  Also cudaErrorInvalidValue, without a launch, for a null map or n_groups outside 1..64; the ids
// themselves are checked on the host where the map is built.
int b2_adamw_flat_grouped_launch(float* p, float* m, float* v, float* g, size_t n, const uint8_t* map, const b2::AdamwScalars* s,
                                 const b2::AdamwGroups* gs, int n_groups, int zero_grad, float max_norm, const double* sqnorms,
                                 int n_buckets, float* grad_norm_out, const float* grad_scale, cudaStream_t stream) {
  if (p == nullptr || m == nullptr || v == nullptr || g == nullptr || s == nullptr || map == nullptr || gs == nullptr ||
      n_groups < 1 || n_groups > b2::kMaxGroups)
    return (int)cudaErrorInvalidValue;
  const size_t n4 = (n / 4) > 0 ? n / 4 : 1;
  const unsigned blocks = (unsigned)((n4 + 255) / 256);
  using namespace b2;
  const bool scaled = grad_scale != nullptr;
  if (max_norm > 0.f) {
    if (sqnorms == nullptr || n_buckets < 1 || !(max_norm < INFINITY)) return (int)cudaErrorInvalidValue;
    if (scaled)
      adamw_flat_grouped_kernel<true, true><<<blocks, 256, 0, stream>>>(p, m, v, g, n, map, *s, *gs, zero_grad, sqnorms, n_buckets,
                                                                        max_norm, grad_norm_out, grad_scale);
    else
      adamw_flat_grouped_kernel<true, false><<<blocks, 256, 0, stream>>>(p, m, v, g, n, map, *s, *gs, zero_grad, sqnorms, n_buckets,
                                                                         max_norm, grad_norm_out, nullptr);
  } else if (scaled) {
    adamw_flat_grouped_kernel<false, true><<<blocks, 256, 0, stream>>>(p, m, v, g, n, map, *s, *gs, zero_grad, nullptr, 0, 0.f,
                                                                       nullptr, grad_scale);
  } else {
    adamw_flat_grouped_kernel<false, false><<<blocks, 256, 0, stream>>>(p, m, v, g, n, map, *s, *gs, zero_grad, nullptr, 0, 0.f,
                                                                        nullptr, nullptr);
  }
  return (int)cudaGetLastError();
}

}  // extern "C"
