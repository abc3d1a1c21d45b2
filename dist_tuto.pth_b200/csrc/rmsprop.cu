// FlatRMSprop's update of one gradient bucket on sm_90a (ops/optim.py): RMSprop over the flat fp32 parameters, the square
// average (and, when they exist, the momentum buffer and the centered gradient average) and the averaged gradients, one launch
// per bucket, streaming every array once and re-zeroing the gradients in the same pass.  The per-element sequence is
// rmsprop_elem (rmsprop_device.cuh).
#include <cstring>
#include "flat_scalars.cuh"
#include "param_groups.cuh"
#include "rmsprop_device.cuh"
#include "sgd_device.cuh"

namespace b2 {

// Everything one launch reads.  `ga` / `buf` are null when the update is not centered / has no momentum (s.centered and
// s.momentum say the same).  `gs` (by value): the groups' lr and weight decay of the grouped, non-capturable instances.
struct RmspropFlatArgs {
  float* p;
  float* sq;
  float* ga;
  float* buf;
  float* g;
  size_t n;
  const uint8_t* map;           // one group id per parameter vector (grouped instances)
  const FlatScalars* blk;       // capturable instances: lr / wd (and every group's) from the device block
  RmspropScalars s;
  SgdGroups gs;
  int zero_grad;
  const double* sqnorms;        // clip instances: grad_sqnorm's per-bucket sums
  int n_buckets;
  float max_norm;
  float* grad_norm_out;
  const float* grad_scale;      // scaled instances: GradScaler's loss scale
  const float* found_inf;       // capturable scaled instances: GradScaler's skip flag
};

// One kernel for every instance, as adamw.cu's three kernels are per instance:
//   kClip     g *= coef first, coef = clip_coef(total norm), the norm sqrt(sum of sqnorms) in fp64 rounded once;
//   kScaled   the gradient is g * amp_inv_scale(grad_scale) (sgd_device.cuh), unscaled before the clip coefficient; with
//             kCap also GradScaler's skip: found_inf != 0 writes only the zeroing, and a null grad_scale means already
//             unscaled;
//   kGrouped  parameter vector i takes lr and weight decay of group map[i]; the tail (< 4 elements) shares the map entry of
//             its vector;
//   kCap      lr and weight decay (kGrouped: every group's) come from the scalar block `blk` on the device (flat_scalars.cuh),
//             loaded once per CTA through shared memory; alpha, 1 - alpha, eps and momentum come from the arguments.
// The per-element code is rmsprop_elem in every instance, so the same scalars give the same bits.
template <bool kClip, bool kGrouped, bool kScaled, bool kCap>
__global__ void __launch_bounds__(256) rmsprop_flat_kernel(const RmspropFlatArgs a) {
  __shared__ float s_coef;
  __shared__ float s_lr, s_wd;
  __shared__ SgdGroups s_gs;
  if constexpr (kCap && kScaled) {
    if (__ldg(a.found_inf) != 0.f) {
      amp_skip_zero(a.g, a.n, a.zero_grad);
      return;
    }
  }
  if constexpr (kCap) {
    if constexpr (kGrouped) flat_block_load(s_gs, a.blk->sgd);
    else if (threadIdx.x == 0) { s_lr = __ldg(&a.blk->lr); s_wd = __ldg(&a.blk->wd); }
  }
  if constexpr (kClip) {
    if (threadIdx.x == 0) s_coef = flat_clip_coef(a.sqnorms, a.n_buckets, a.max_norm, a.grad_norm_out);
  }
  if constexpr (kCap || kClip) __syncthreads();
  const float c = kClip ? s_coef : 1.f;
  RmspropScalars s = a.s;
  if constexpr (kCap && !kGrouped) { s.lr = s_lr; s.wd = s_wd; }
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n4 = a.n / 4;
  const float inv = kScaled && (!kCap || a.grad_scale != nullptr) ? amp_inv_scale(a.grad_scale) : 1.f;
  if (i < n4) {
    if constexpr (kGrouped) {
      const int gid = a.map[i];
      if constexpr (kCap) { s.lr = s_gs.lr[gid]; s.wd = s_gs.wd[gid]; }
      else { s.lr = a.gs.lr[gid]; s.wd = a.gs.wd[gid]; }
    }
    float4 gv = reinterpret_cast<const float4*>(a.g)[i];
    float4 pv = reinterpret_cast<float4*>(a.p)[i];
    float4 sv = reinterpret_cast<float4*>(a.sq)[i];
    float4 av = make_float4(0.f, 0.f, 0.f, 0.f), bv = av;
    if (s.centered) av = reinterpret_cast<float4*>(a.ga)[i];
    if (s.momentum) bv = reinterpret_cast<float4*>(a.buf)[i];
    if constexpr (kScaled) gv = amp_unscale4(gv, inv);
    if constexpr (kClip) {
      gv.x = __fmul_rn(gv.x, c); gv.y = __fmul_rn(gv.y, c); gv.z = __fmul_rn(gv.z, c); gv.w = __fmul_rn(gv.w, c);
    }
    rmsprop4(pv, sv, av, bv, gv, s);
    reinterpret_cast<float4*>(a.p)[i] = pv;
    reinterpret_cast<float4*>(a.sq)[i] = sv;
    if (s.centered) reinterpret_cast<float4*>(a.ga)[i] = av;
    if (s.momentum) reinterpret_cast<float4*>(a.buf)[i] = bv;
    if (a.zero_grad) reinterpret_cast<float4*>(a.g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (i < a.n - n4 * 4) {                      // tail (< 4 elements): threads 0..2 of CTA 0, one element each
    const size_t t = n4 * 4 + i;
    if constexpr (kGrouped) {
      const int gid = a.map[n4];
      if constexpr (kCap) { s.lr = s_gs.lr[gid]; s.wd = s_gs.wd[gid]; }
      else { s.lr = a.gs.lr[gid]; s.wd = a.gs.wd[gid]; }
    }
    const float gl = kScaled ? amp_unscale(a.g[t], inv) : a.g[t];
    const float gt = kClip ? __fmul_rn(gl, c) : gl;
    float ga = 0.f, buf = 0.f;
    if (s.centered) ga = a.ga[t];
    if (s.momentum) buf = a.buf[t];
    rmsprop_elem(a.p[t], a.sq[t], ga, buf, gt, s);
    if (s.centered) a.ga[t] = ga;
    if (s.momentum) a.buf[t] = buf;
    if (a.zero_grad) a.g[t] = 0.f;
  }
}

}  // namespace b2

extern "C" {

// One RMSprop update of a flat bucket of n elements on `stream`.  s: the update's scalars (s->centered / s->momentum are set
// here from ga / buf).  map: null without groups, else one group id per parameter vector, with gs holding n_groups groups'
// lr and weight decay.  blk: null for the eager instances, else the capturable ones (lr / wd from the block, gs unused).
// max_norm > 0: clipped by the norm of grad_sqnorm's n_buckets sums.  grad_scale: GradScaler's loss scale (or null); found_inf
// (capturable only): GradScaler's skip flag.  cudaErrorInvalidValue, without a launch, for a null pointer, clipping without
// sqnorms, n_groups outside 1..64 with a map, found_inf without a block or grad_scale without found_inf on the block path.
int b2_rmsprop_flat_launch(float* p, float* sq, float* ga, float* buf, float* g, size_t n, const uint8_t* map,
                           const b2::RmspropScalars* s, const b2::SgdGroups* gs, int n_groups, const b2::FlatScalars* blk,
                           int zero_grad, float max_norm, const double* sqnorms, int n_buckets, float* grad_norm_out,
                           const float* grad_scale, const float* found_inf, cudaStream_t stream) {
  using namespace b2;
  if (p == nullptr || sq == nullptr || g == nullptr || s == nullptr) return (int)cudaErrorInvalidValue;
  const bool cap = blk != nullptr, grouped = map != nullptr, clip = max_norm > 0.f;
  if (grouped && !cap && (gs == nullptr || n_groups < 1 || n_groups > kMaxGroups)) return (int)cudaErrorInvalidValue;
  if (clip && (sqnorms == nullptr || n_buckets < 1 || !(max_norm < INFINITY))) return (int)cudaErrorInvalidValue;
  if (cap ? (found_inf == nullptr && grad_scale != nullptr) : found_inf != nullptr) return (int)cudaErrorInvalidValue;
  RmspropFlatArgs a;
  memset(&a, 0, sizeof(a));
  a.p = p; a.sq = sq; a.ga = ga; a.buf = buf; a.g = g; a.n = n; a.map = map; a.blk = blk;
  a.s = *s;
  a.s.centered = ga != nullptr ? 1 : 0;
  a.s.momentum = buf != nullptr ? 1 : 0;
  if (grouped && !cap) a.gs = *gs;
  a.zero_grad = zero_grad;
  if (clip) { a.sqnorms = sqnorms; a.n_buckets = n_buckets; a.max_norm = max_norm; a.grad_norm_out = grad_norm_out; }
  a.grad_scale = grad_scale;
  a.found_inf = found_inf;
  const size_t n4 = (n / 4) > 0 ? n / 4 : 1;
  const unsigned blocks = (unsigned)((n4 + 255) / 256);
  const bool scaled = cap ? found_inf != nullptr : grad_scale != nullptr;
#define B2_RMSPROP(C, G, S, K) rmsprop_flat_kernel<C, G, S, K><<<blocks, 256, 0, stream>>>(a)
  const int k = (cap ? 8 : 0) | (scaled ? 4 : 0) | (clip ? 2 : 0) | (grouped ? 1 : 0);
  switch (k) {
    case 0: B2_RMSPROP(false, false, false, false); break;
    case 1: B2_RMSPROP(false, true, false, false); break;
    case 2: B2_RMSPROP(true, false, false, false); break;
    case 3: B2_RMSPROP(true, true, false, false); break;
    case 4: B2_RMSPROP(false, false, true, false); break;
    case 5: B2_RMSPROP(false, true, true, false); break;
    case 6: B2_RMSPROP(true, false, true, false); break;
    case 7: B2_RMSPROP(true, true, true, false); break;
    case 8: B2_RMSPROP(false, false, false, true); break;
    case 9: B2_RMSPROP(false, true, false, true); break;
    case 10: B2_RMSPROP(true, false, false, true); break;
    case 11: B2_RMSPROP(true, true, false, true); break;
    case 12: B2_RMSPROP(false, false, true, true); break;
    case 13: B2_RMSPROP(false, true, true, true); break;
    case 14: B2_RMSPROP(true, false, true, true); break;
    default: B2_RMSPROP(true, true, true, true); break;
  }
#undef B2_RMSPROP
  return (int)cudaGetLastError();
}

}  // extern "C"
