// FlatLAMB's and FlatLARS's update of one fp32 gradient bucket on sm_90a (ops/optim.py): per-tensor trust ratios from
// per-tensor norms over the flat bucket, in two launches and without a host synchronisation.
//
//   layerwise_norms_kernel   per chunk of the table (layerwise.h): LAMB updates m and v and forms u; both sum p^2 and
//                            u^2 (LAMB) or g^2 (LARS) per thread in fp32 (fmaf, the thread's float4 vectors in order, then
//                            its tail element), per CTA in a fixed tree, and write the two chunk partials.  The last CTA to
//                            finish a tensor (per-tensor ticket) adds the tensor's partials in chunk order in fp64.
//   layerwise_apply_kernel   the same chunks: the ratio from the tensor's two sums (fp64, rounded once to fp32), then
//                            LAMB p -= (lr * r) * u with u recomputed from the stored moments, or LARS's momentum step on
//                            d = r * (g + wd * p); the gradients re-zeroed.
// The order of every sum depends on the table only, never on the grid or on timing, so two runs are bit-identical.
#include "layerwise_device.cuh"
#include "sgd_device.cuh"

namespace b2 {

constexpr int kLwMaxCtas = 2048;     // grid-stride over the chunks beyond this

// The clip coefficient of grad_sqnorm's sums, as adamw_flat_kernel<true> takes it; CTA 0 of the norms kernel writes the norm.
__device__ __forceinline__ float lw_clip_coef(const LwArgs& a, bool write_norm) {
  __shared__ float s_coef;
  if (threadIdx.x == 0) {
    double q = 0.0;
    for (int k = 0; k < a.n_buckets; ++k) q += a.sqnorms[k];
    const float nrm = __double2float_rn(__dsqrt_rn(q));
    s_coef = clip_coef(nrm, a.max_norm);
    if (write_norm && blockIdx.x == 0 && a.grad_norm_out != nullptr) *a.grad_norm_out = nrm;
  }
  __syncthreads();
  return s_coef;
}

__device__ __forceinline__ float4 scale4(float4 g, float c) {
  return make_float4(__fmul_rn(g.x, c), __fmul_rn(g.y, c), __fmul_rn(g.z, c), __fmul_rn(g.w, c));
}

// kScaled: every gradient is read as g * amp_inv_scale(a.grad_scale) (sgd_device.cuh), before the clip coefficient.
template <bool kLamb, bool kClip, bool kScaled>
__global__ void __launch_bounds__(kLwThreads) layerwise_norms_kernel(const LwArgs a) {
  __shared__ float2 s_warp[kLwThreads / 32];
  __shared__ float2 s_stage[kLwThreads];
  __shared__ int s_last;
  float c = 1.f;
  if constexpr (kClip) c = lw_clip_coef(a, true);
  const float inv = kScaled ? amp_inv_scale(a.grad_scale) : 1.f;
  const long long* chunks = a.table;
  const long long* tens = a.table + (size_t)a.n_chunks * kLwRow;
  for (int ch = blockIdx.x; ch < a.n_chunks; ch += gridDim.x) {
    const long long start = chunks[ch * kLwRow], len = chunks[ch * kLwRow + 1];
    const int t = (int)chunks[ch * kLwRow + 2];
    const float wd = kLamb && tens[t * kLwRow + 2] != 0 ? a.wd : 0.f;
    const int nv = (int)(len >> 2), tail = (int)(len & 3);
    const size_t v0 = (size_t)start >> 2;
    float sp = 0.f, sq = 0.f;
#pragma unroll 4
    for (int i = threadIdx.x; i < nv; i += kLwThreads) {
      const float4 pv = reinterpret_cast<const float4*>(a.p)[v0 + i];
      float4 gv = reinterpret_cast<const float4*>(a.g)[v0 + i];
      if constexpr (kScaled) gv = amp_unscale4(gv, inv);
      if constexpr (kClip) gv = scale4(gv, c);
      sp = fmaf(pv.x, pv.x, sp); sp = fmaf(pv.y, pv.y, sp); sp = fmaf(pv.z, pv.z, sp); sp = fmaf(pv.w, pv.w, sp);
      if constexpr (kLamb) {
        float4 mv = reinterpret_cast<const float4*>(a.m)[v0 + i];
        float4 vv = reinterpret_cast<const float4*>(a.v)[v0 + i];
        adam_moments(mv.x, vv.x, gv.x, a);
        adam_moments(mv.y, vv.y, gv.y, a);
        adam_moments(mv.z, vv.z, gv.z, a);
        adam_moments(mv.w, vv.w, gv.w, a);
        reinterpret_cast<float4*>(a.m)[v0 + i] = mv;
        reinterpret_cast<float4*>(a.v)[v0 + i] = vv;
        const float ux = lamb_u(pv.x, mv.x, vv.x, wd, a), uy = lamb_u(pv.y, mv.y, vv.y, wd, a);
        const float uz = lamb_u(pv.z, mv.z, vv.z, wd, a), uw = lamb_u(pv.w, mv.w, vv.w, wd, a);
        sq = fmaf(ux, ux, sq); sq = fmaf(uy, uy, sq); sq = fmaf(uz, uz, sq); sq = fmaf(uw, uw, sq);
      } else {
        sq = fmaf(gv.x, gv.x, sq); sq = fmaf(gv.y, gv.y, sq); sq = fmaf(gv.z, gv.z, sq); sq = fmaf(gv.w, gv.w, sq);
      }
    }
    if (threadIdx.x < tail) {                  // a tensor's last < 4 elements: threads 0..2, one each
      const size_t e = (size_t)start + (size_t)nv * 4 + threadIdx.x;
      const float pe = a.p[e];
      const float gl = kScaled ? amp_unscale(a.g[e], inv) : a.g[e];
      const float ge = kClip ? __fmul_rn(gl, c) : gl;
      sp = fmaf(pe, pe, sp);
      if constexpr (kLamb) {
        float me = a.m[e], ve = a.v[e];
        adam_moments(me, ve, ge, a);
        a.m[e] = me;
        a.v[e] = ve;
        const float u = lamb_u(pe, me, ve, wd, a);
        sq = fmaf(u, u, sq);
      } else {
        sq = fmaf(ge, ge, sq);
      }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      sp += __shfl_xor_sync(0xffffffffu, sp, d);
      sq += __shfl_xor_sync(0xffffffffu, sq, d);
    }
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = make_float2(sp, sq);
    __syncthreads();
    const long long first = tens[t * kLwRow], cnt = tens[t * kLwRow + 1];
    if (threadIdx.x == 0) {
      float tp = 0.f, tq = 0.f;
      for (int w = 0; w < kLwThreads / 32; ++w) {
        tp += s_warp[w].x;
        tq += s_warp[w].y;
      }
      __stcg(reinterpret_cast<float2*>(a.partials) + ch, make_float2(tp, tq));
      __threadfence();
      s_last = atomicAdd(a.tickets + t, 1u) == (unsigned int)(cnt - 1);
      if (s_last) __threadfence();
    }
    __syncthreads();
    if (s_last) {                              // uniform: the tensor's partials, in chunk order, in fp64
      double dp = 0.0, dq = 0.0;
      for (long long b = 0; b < cnt; b += kLwThreads) {
        if (b + threadIdx.x < cnt) s_stage[threadIdx.x] = __ldcg(reinterpret_cast<const float2*>(a.partials) + first + b + threadIdx.x);
        __syncthreads();
        if (threadIdx.x == 0) {
          const int k_end = cnt - b < kLwThreads ? (int)(cnt - b) : kLwThreads;
          for (int k = 0; k < k_end; ++k) {
            dp = __dadd_rn(dp, (double)s_stage[k].x);
            dq = __dadd_rn(dq, (double)s_stage[k].y);
          }
        }
        __syncthreads();
      }
      if (threadIdx.x == 0) {
        a.sums[2 * t] = dp;
        a.sums[2 * t + 1] = dq;
        a.tickets[t] = 0u;
      }
    }
  }
}

template <bool kLamb, bool kClip, bool kScaled>
__global__ void __launch_bounds__(kLwThreads) layerwise_apply_kernel(const LwArgs a) {
  __shared__ float s_r;
  float c = 1.f;
  if constexpr (kClip) c = lw_clip_coef(a, false);
  const float inv = kScaled ? amp_inv_scale(a.grad_scale) : 1.f;
  const long long* chunks = a.table;
  const long long* tens = a.table + (size_t)a.n_chunks * kLwRow;
  for (int ch = blockIdx.x; ch < a.n_chunks; ch += gridDim.x) {
    const long long start = chunks[ch * kLwRow], len = chunks[ch * kLwRow + 1];
    const int t = (int)chunks[ch * kLwRow + 2];
    const bool adapt = tens[t * kLwRow + 2] != 0;
    __syncthreads();                           // the previous chunk's readers of s_r are done
    if (threadIdx.x == 0) {
      const double w = __dsqrt_rn(a.sums[2 * t]), q = __dsqrt_rn(a.sums[2 * t + 1]);
      float r = 1.f;
      if (adapt && w > 0.0 && q > 0.0)
        r = kLamb ? __double2float_rn(__ddiv_rn(w, q))
                  : __double2float_rn(__ddiv_rn(__dmul_rn(a.eta64, w), __dadd_rn(__dadd_rn(q, __dmul_rn(a.wd64, w)), a.eps64)));
      s_r = r;
      if (ch == (int)tens[t * kLwRow]) a.ratios[t] = r;
    }
    __syncthreads();
    const float r = s_r;
    const float wd = adapt ? a.wd : 0.f;
    const int nv = (int)(len >> 2), tail = (int)(len & 3);
    const size_t v0 = (size_t)start >> 2;
    if constexpr (kLamb) {
      const float step = -__fmul_rn(a.lr, r);
#pragma unroll 4
      for (int i = threadIdx.x; i < nv; i += kLwThreads) {
        float4 pv = reinterpret_cast<const float4*>(a.p)[v0 + i];
        const float4 mv = reinterpret_cast<const float4*>(a.m)[v0 + i];
        const float4 vv = reinterpret_cast<const float4*>(a.v)[v0 + i];
        pv.x = fmaf(step, lamb_u(pv.x, mv.x, vv.x, wd, a), pv.x);
        pv.y = fmaf(step, lamb_u(pv.y, mv.y, vv.y, wd, a), pv.y);
        pv.z = fmaf(step, lamb_u(pv.z, mv.z, vv.z, wd, a), pv.z);
        pv.w = fmaf(step, lamb_u(pv.w, mv.w, vv.w, wd, a), pv.w);
        reinterpret_cast<float4*>(a.p)[v0 + i] = pv;
        if (a.zero_grad) reinterpret_cast<float4*>(a.g)[v0 + i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      if (threadIdx.x < tail) {
        const size_t e = (size_t)start + (size_t)nv * 4 + threadIdx.x;
        a.p[e] = fmaf(step, lamb_u(a.p[e], a.m[e], a.v[e], wd, a), a.p[e]);
        if (a.zero_grad) a.g[e] = 0.f;
      }
    } else {
#pragma unroll 4
      for (int i = threadIdx.x; i < nv; i += kLwThreads) {
        float4 pv = reinterpret_cast<const float4*>(a.p)[v0 + i];
        float4 mv = reinterpret_cast<const float4*>(a.m)[v0 + i];
        float4 gv = reinterpret_cast<const float4*>(a.g)[v0 + i];
        if constexpr (kScaled) gv = amp_unscale4(gv, inv);
        if constexpr (kClip) gv = scale4(gv, c);
        lars_elem(pv.x, mv.x, gv.x, r, wd, a);
        lars_elem(pv.y, mv.y, gv.y, r, wd, a);
        lars_elem(pv.z, mv.z, gv.z, r, wd, a);
        lars_elem(pv.w, mv.w, gv.w, r, wd, a);
        reinterpret_cast<float4*>(a.p)[v0 + i] = pv;
        reinterpret_cast<float4*>(a.m)[v0 + i] = mv;
        if (a.zero_grad) reinterpret_cast<float4*>(a.g)[v0 + i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      if (threadIdx.x < tail) {
        const size_t e = (size_t)start + (size_t)nv * 4 + threadIdx.x;
        float pe = a.p[e], me = a.m[e];
        const float gl = kScaled ? amp_unscale(a.g[e], inv) : a.g[e];
        lars_elem(pe, me, kClip ? __fmul_rn(gl, c) : gl, r, wd, a);
        a.p[e] = pe;
        a.m[e] = me;
        if (a.zero_grad) a.g[e] = 0.f;
      }
    }
  }
}

template <bool kLamb, bool kClip, bool kScaled>
int layerwise_launch_t(const LwArgs& a, cudaStream_t stream) {
  const unsigned blocks = (unsigned)(a.n_chunks < kLwMaxCtas ? a.n_chunks : kLwMaxCtas);
  layerwise_norms_kernel<kLamb, kClip, kScaled><<<blocks, kLwThreads, 0, stream>>>(a);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  // LAMB's second pass does not read g, so it has no clip or scaled instance
  layerwise_apply_kernel<kLamb, kClip && !kLamb, kScaled && !kLamb><<<blocks, kLwThreads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

}  // namespace b2

extern "C" {

// One FlatLAMB (lamb != 0) or FlatLARS update of a flat bucket on `stream`: the norms kernel, then the apply kernel.
// max_norm > 0: g is clipped by the norm of grad_sqnorm's n_buckets sums.  cudaErrorInvalidValue, without a launch, for a
// null pointer, an empty or inconsistent table, or clipping without sqnorms.  The bindings check the table's rows.
int b2_layerwise_launch(int lamb, const b2::LwArgs* a, cudaStream_t stream) {
  if (a == nullptr || a->p == nullptr || a->g == nullptr || a->m == nullptr || (lamb && a->v == nullptr) || a->table == nullptr ||
      a->partials == nullptr || a->tickets == nullptr || a->sums == nullptr || a->ratios == nullptr)
    return (int)cudaErrorInvalidValue;
  if (a->n_tensors < 1 || a->n_chunks < 1 || (size_t)a->n_chunks > a->n) return (int)cudaErrorInvalidValue;
  const bool clip = a->max_norm > 0.f;
  if (clip && (a->sqnorms == nullptr || a->n_buckets < 1 || !(a->max_norm < INFINITY))) return (int)cudaErrorInvalidValue;
  using namespace b2;
  const int k = (lamb ? 4 : 0) | (clip ? 2 : 0) | (a->grad_scale != nullptr ? 1 : 0);
  switch (k) {
    case 0: return layerwise_launch_t<false, false, false>(*a, stream);
    case 1: return layerwise_launch_t<false, false, true>(*a, stream);
    case 2: return layerwise_launch_t<false, true, false>(*a, stream);
    case 3: return layerwise_launch_t<false, true, true>(*a, stream);
    case 4: return layerwise_launch_t<true, false, false>(*a, stream);
    case 5: return layerwise_launch_t<true, false, true>(*a, stream);
    case 6: return layerwise_launch_t<true, true, false>(*a, stream);
    default: return layerwise_launch_t<true, true, true>(*a, stream);
  }
}

}  // extern "C"
