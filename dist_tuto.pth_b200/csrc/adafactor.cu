// FlatAdafactor's update of one fp32 gradient bucket on sm_90a (ops/optim.py): torch.optim.Adafactor's factored second
// moments and per-tensor step sizes, in three launches over the chunk table of adafactor.h and without a host
// synchronisation.  Update t of a tensor (w = fp32(t ** beta2_decay), rho = min(lr, 1 / sqrt(t)), lr the scheduled lr):
//
//   adafactor_stats_kernel  per chunk: the sum of p^2 (fp32: fmaf per thread over the box in logical order, xor
//                           butterflies, the warps in order), and
//                           unfactored: variance = lerp(variance, g*g, w);
//                           factored:   the chunk's gradients staged in shared memory; per row and per column of the box
//                           one thread adds g^2 in order (fmaf, fp32).  A whole-slice chunk then lerps row_var / col_var
//                           towards fp32(sqrt(sum))^2 / C (/ R) and forms every slice's clamped row_var mean; a tile writes
//                           its row and column partials instead.
//                           The tensor's last CTA (per-tensor ticket) adds the p^2 partials in chunk order in fp64, forms
//                           alpha = max(eps2, fp32(||p||) / sqrt(numel)) * rho in fp64, and for a tiled tensor adds each
//                           row's and column's partials in tile order in fp64, lerps, and forms the slices' means.
//   adafactor_norm_kernel   per chunk: u = (1 / sqrt(max(v, eps1^2))) * g with v = fp32(row_var * col_var) / mean (or
//                           the variance); the sum of u^2 as above.  The last CTA: ||u|| in fp64 from the partials in chunk
//                           order, rounded to fp32; step = fp32(-alpha / max(1, ||u|| / (sqrt(numel) * d))).
//   adafactor_apply_kernel  per chunk: p = fmaf(step, u, p * fp32(1 - lr * wd)) with u recomputed; g re-zeroed.
// A slice's row_var mean adds its rows in blocks of ceil(R / 256) rows: fp64 in row order within a block, then the blocks in
// order, divided by R in fp64 and rounded once.  The order of every sum depends on the table only, never on the grid or on
// timing, and no sum uses an atomic, so two runs are bit-identical.  tests/adafactor_model.py is the same sequence on the CPU.
#include "adafactor.h"
#include "sgd_device.cuh"

namespace b2 {

constexpr int kAfMaxCtas = 2048;     // grid-stride over the chunks beyond this

// The clip coefficient of grad_sqnorm's sums; CTA 0 of the stats kernel writes the norm.
__device__ __forceinline__ float af_clip_coef(const AfArgs& a, bool write_norm) {
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

// The gradient the update reads: unscaled (GradScaler), then clipped.
template <bool kClip, bool kScaled>
__device__ __forceinline__ float af_grad(float g, float inv, float c) {
  if constexpr (kScaled) g = amp_unscale(g, inv);
  if constexpr (kClip) g = __fmul_rn(g, c);
  return g;
}

// torch's lerp: s + w * (e - s) for w < 0.5, else e - (e - s) * (1 - w), each as one fused multiply-add
__device__ __forceinline__ float af_lerp(float s, float e, float w) {
  const float d = __fsub_rn(e, s);
  return w < 0.5f ? fmaf(w, d, s) : fmaf(__fsub_rn(w, 1.f), d, e);
}

// torch's row / column mean of g^2: the fp32 norm from the fp64 sum of squares, squared in fp32, divided by the count
__device__ __forceinline__ float af_sq_mean(double s, float n) {
  const float nrm = __double2float_rn(__dsqrt_rn(s));
  return __fdiv_rn(__fmul_rn(nrm, nrm), n);
}

// u = rsqrt(clamp(v, eps1^2)) * g, the root and the reciprocal rounded separately; a NaN passes the clamp
__device__ __forceinline__ float af_u(float v, float g, float eps1sq) {
  const float c = v < eps1sq ? eps1sq : v;
  return __fmul_rn(__fdiv_rn(1.f, __fsqrt_rn(c)), g);
}

__device__ __forceinline__ float af_clamp_mean(double s, long long R, float eps1) {
  const float m = __double2float_rn(__ddiv_rn(s, (double)R));
  return m < eps1 ? eps1 : m;
}

// The offset of slice b from its leading sizes and strides (row-major over the leading dimensions)
__device__ __forceinline__ long long af_lead(const long long* T, unsigned b) {
  const int nl = (int)T[AF_NLEAD];
  if (nl == 0) return 0;
  if (nl == 1) return (long long)b * T[AF_LSTRIDE];
  long long off = 0;
  for (int k = nl - 1; k >= 0; --k) {
    const unsigned s = (unsigned)T[AF_LSIZE + k];
    off += (long long)(b % s) * T[AF_LSTRIDE + k];
    b /= s;
  }
  return off;
}

// One chunk of the table, with its tensor's row
struct AfBox {
  const long long* T;
  int t;
  long long b0, r0, c0;
  unsigned nb, nr, nc;
};
__device__ __forceinline__ AfBox af_box(const AfArgs& a, int ch) {
  const long long* row = a.table + (size_t)ch * kAfChunkRow;
  AfBox x;
  x.t = (int)row[0];
  x.T = a.table + (size_t)a.n_chunks * kAfChunkRow + (size_t)x.t * kAfTensorRow;
  x.b0 = row[1]; x.nb = (unsigned)row[2]; x.r0 = row[3]; x.nr = (unsigned)row[4]; x.c0 = row[5]; x.nc = (unsigned)row[6];
  return x;
}
// Element j of the box (logical order, columns fastest): its (slice, row, column) relative to the box and its flat index
struct AfElem {
  unsigned bi, ri, ci;
  size_t e;
};
__device__ __forceinline__ AfElem af_elem(const AfBox& x, unsigned j) {
  AfElem r;
  r.ci = j % x.nc;
  const unsigned q = j / x.nc;
  r.ri = q % x.nr;
  r.bi = q / x.nr;
  const long long* T = x.T;
  r.e = (size_t)(T[AF_OFFSET] + af_lead(T, (unsigned)(x.b0 + r.bi)) + (x.r0 + r.ri) * T[AF_SR] + (x.c0 + r.ci) * T[AF_SC]);
  return r;
}
// v of an element: fp32(row_var * col_var) / mean, or the variance
__device__ __forceinline__ float af_v(const AfArgs& a, const AfBox& x, const AfElem& el) {
  const long long* T = x.T;
  const float* st = a.state + T[AF_STATE];
  if (T[AF_FACTORED] == 0) return st[x.c0 + el.ci];
  const long long b = x.b0 + el.bi, B = T[AF_B], R = T[AF_R], C = T[AF_C];
  return __fdiv_rn(__fmul_rn(st[b * R + x.r0 + el.ri], st[B * R + b * C + x.c0 + el.ci]), a.means[T[AF_MEAN] + b]);
}

// The CTA's fp32 sum of the threads' values: xor butterflies in each warp, then the warps in order (thread 0's result).
__device__ __forceinline__ float af_cta_sum(float s, float* s_warp) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = s;
  __syncthreads();
  float tot = 0.f;
  if (threadIdx.x == 0)
    for (int w = 0; w < kAfThreads / 32; ++w) tot += s_warp[w];
  return tot;
}

// Thread 0 stores the chunk's partial and takes the tensor's ticket; true in every thread of the tensor's last CTA, which
// then sees every partial and state the tensor's CTAs wrote.  Every thread fences its own writes first.
__device__ __forceinline__ bool af_ticket(const AfArgs& a, float* slot, float tot, int t, long long cnt, int* s_last) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    __stcg(slot, tot);
    __threadfence();
    *s_last = atomicAdd(a.tickets + t, 1u) == (unsigned int)(cnt - 1);
    if (*s_last) __threadfence();
  }
  __syncthreads();
  return *s_last != 0;
}

// The fp64 sum of a tensor's chunk partials part[first, first + cnt), in chunk order (thread 0)
__device__ __forceinline__ double af_chunk_sum(const float* part, long long first, long long cnt) {
  double s = 0.0;
  for (long long k = 0; k < cnt; ++k) s = __dadd_rn(s, (double)__ldcg(part + first + k));
  return s;
}

template <bool kClip, bool kScaled>
__global__ void __launch_bounds__(kAfThreads) adafactor_stats_kernel(const AfArgs a) {
  extern __shared__ float s_g[];
  __shared__ float s_warp[kAfThreads / 32];
  __shared__ double s_d[kAfThreads];
  __shared__ int s_last;
  float c = 1.f;
  if constexpr (kClip) c = af_clip_coef(a, true);
  const float inv = kScaled ? amp_inv_scale(a.grad_scale) : 1.f;
  for (int ch = blockIdx.x; ch < a.n_chunks; ch += gridDim.x) {
    const AfBox x = af_box(a, ch);
    const long long* T = x.T;
    const bool fac = T[AF_FACTORED] != 0, whole = T[AF_WHOLE] != 0;
    const long long B = T[AF_B], R = T[AF_R], C = T[AF_C];
    float* st = a.state + T[AF_STATE];
    const unsigned L = x.nb * x.nr * x.nc, pitch = x.nc | 1u;
    __syncthreads();                           // the previous chunk's readers of s_g are done
    float sp = 0.f;
    for (unsigned j = threadIdx.x; j < L; j += kAfThreads) {
      const AfElem el = af_elem(x, j);
      const float pe = a.p[el.e];
      const float ge = af_grad<kClip, kScaled>(a.g[el.e], inv, c);
      sp = fmaf(pe, pe, sp);
      if (fac) {
        s_g[(el.bi * x.nr + el.ri) * pitch + el.ci] = ge;
      } else {
        const long long k = x.c0 + el.ci;
        st[k] = af_lerp(st[k], __fmul_rn(ge, ge), a.w);
      }
    }
    if (fac) {
      __syncthreads();
      const long long ntc = whole ? 1 : (C + T[AF_TC] - 1) / T[AF_TC], ntr = whole ? 1 : (R + T[AF_TR] - 1) / T[AF_TR];
      float* rcp = a.rc + T[AF_RC];
      for (unsigned i = threadIdx.x; i < x.nb * x.nr; i += kAfThreads) {
        float s = 0.f;
        for (unsigned k = 0; k < x.nc; ++k) {
          const float ge = s_g[i * pitch + k];
          s = fmaf(ge, ge, s);
        }
        const long long b = x.b0 + i / x.nr, r = x.r0 + i % x.nr;
        if (whole) st[b * R + r] = af_lerp(st[b * R + r], af_sq_mean((double)s, (float)C), a.w);
        else __stcg(rcp + (b * R + r) * ntc + x.c0 / T[AF_TC], s);
      }
      for (unsigned i = threadIdx.x; i < x.nb * x.nc; i += kAfThreads) {
        const unsigned bi = i / x.nc, ci = i % x.nc;
        float s = 0.f;
        for (unsigned k = 0; k < x.nr; ++k) {
          const float ge = s_g[(bi * x.nr + k) * pitch + ci];
          s = fmaf(ge, ge, s);
        }
        const long long b = x.b0 + bi, cc = x.c0 + ci;
        if (whole) st[B * R + b * C + cc] = af_lerp(st[B * R + b * C + cc], af_sq_mean((double)s, (float)R), a.w);
        else __stcg(rcp + B * R * ntc + (b * C + cc) * ntr + x.r0 / T[AF_TR], s);
      }
      if (whole) {
        __syncthreads();
        for (unsigned bi = threadIdx.x; bi < x.nb; bi += kAfThreads) {
          const long long b = x.b0 + bi, blk = (R + kAfThreads - 1) / kAfThreads;
          double s = 0.0;
          for (long long k0 = 0; k0 < R; k0 += blk) {
            double bs = 0.0;
            for (long long r = k0; r < k0 + blk && r < R; ++r) bs = __dadd_rn(bs, (double)st[b * R + r]);
            s = __dadd_rn(s, bs);
          }
          a.means[T[AF_MEAN] + b] = af_clamp_mean(s, R, a.eps1);
        }
      }
    }
    const float tot = af_cta_sum(sp, s_warp);
    if (!af_ticket(a, a.partials + ch, tot, x.t, T[AF_COUNT], &s_last)) continue;
    // the tensor's last CTA
    if (threadIdx.x == 0) {
      const double sq = af_chunk_sum(a.partials, T[AF_FIRST], T[AF_COUNT]);
      const float nrm = __double2float_rn(__dsqrt_rn(sq));
      const double q = __ddiv_rn((double)nrm, __dsqrt_rn((double)(B * R * C)));
      a.alpha[x.t] = __dmul_rn(q > a.eps2 ? q : a.eps2, a.rho[T[AF_GROUP]]);
      a.tickets[x.t] = 0u;
    }
    if (fac && !whole) {
      const long long ntc = (C + T[AF_TC] - 1) / T[AF_TC], ntr = (R + T[AF_TR] - 1) / T[AF_TR];
      const float* rcp = a.rc + T[AF_RC];
      for (long long i = threadIdx.x; i < B * R; i += kAfThreads) {
        double s = 0.0;
        for (long long k = 0; k < ntc; ++k) s = __dadd_rn(s, (double)__ldcg(rcp + i * ntc + k));
        st[i] = af_lerp(st[i], af_sq_mean(s, (float)C), a.w);
      }
      for (long long i = threadIdx.x; i < B * C; i += kAfThreads) {
        double s = 0.0;
        for (long long k = 0; k < ntr; ++k) s = __dadd_rn(s, (double)__ldcg(rcp + B * R * ntc + i * ntr + k));
        st[B * R + i] = af_lerp(st[B * R + i], af_sq_mean(s, (float)R), a.w);
      }
      const long long blk = (R + kAfThreads - 1) / kAfThreads;
      for (long long b = 0; b < B; ++b) {
        __syncthreads();                       // row_var written; s_d free
        const long long k0 = (long long)threadIdx.x * blk;
        double bs = 0.0;
        for (long long r = k0; r < k0 + blk && r < R; ++r) bs = __dadd_rn(bs, (double)st[b * R + r]);
        s_d[threadIdx.x] = bs;
        __syncthreads();
        if (threadIdx.x == 0) {
          double s = 0.0;
          for (long long k = 0; k * blk < R; ++k) s = __dadd_rn(s, s_d[k]);
          a.means[T[AF_MEAN] + b] = af_clamp_mean(s, R, a.eps1);
        }
      }
    }
  }
}

template <bool kClip, bool kScaled>
__global__ void __launch_bounds__(kAfThreads) adafactor_norm_kernel(const AfArgs a) {
  __shared__ float s_warp[kAfThreads / 32];
  __shared__ int s_last;
  float c = 1.f;
  if constexpr (kClip) c = af_clip_coef(a, false);
  const float inv = kScaled ? amp_inv_scale(a.grad_scale) : 1.f;
  for (int ch = blockIdx.x; ch < a.n_chunks; ch += gridDim.x) {
    const AfBox x = af_box(a, ch);
    const long long* T = x.T;
    const unsigned L = x.nb * x.nr * x.nc;
    float su = 0.f;
    for (unsigned j = threadIdx.x; j < L; j += kAfThreads) {
      const AfElem el = af_elem(x, j);
      const float u = af_u(af_v(a, x, el), af_grad<kClip, kScaled>(a.g[el.e], inv, c), a.eps1sq);
      su = fmaf(u, u, su);
    }
    const float tot = af_cta_sum(su, s_warp);
    if (!af_ticket(a, a.partials + a.n_chunks + ch, tot, x.t, T[AF_COUNT], &s_last)) continue;
    if (threadIdx.x == 0) {
      const double sq = af_chunk_sum(a.partials + a.n_chunks, T[AF_FIRST], T[AF_COUNT]);
      const float nrm = __double2float_rn(__dsqrt_rn(sq));
      const double q = __ddiv_rn((double)nrm, __dmul_rn(__dsqrt_rn((double)(T[AF_B] * T[AF_R] * T[AF_C])), a.d));
      a.step[x.t] = __double2float_rn(__ddiv_rn(-a.alpha[x.t], q > 1.0 ? q : 1.0));
      a.tickets[x.t] = 0u;
    }
  }
}

template <bool kClip, bool kScaled>
__global__ void __launch_bounds__(kAfThreads) adafactor_apply_kernel(const AfArgs a) {
  float c = 1.f;
  if constexpr (kClip) c = af_clip_coef(a, false);
  const float inv = kScaled ? amp_inv_scale(a.grad_scale) : 1.f;
  for (int ch = blockIdx.x; ch < a.n_chunks; ch += gridDim.x) {
    const AfBox x = af_box(a, ch);
    const float step = a.step[x.t], decay = a.decay[x.T[AF_GROUP]];
    const unsigned L = x.nb * x.nr * x.nc;
    for (unsigned j = threadIdx.x; j < L; j += kAfThreads) {
      const AfElem el = af_elem(x, j);
      const float u = af_u(af_v(a, x, el), af_grad<kClip, kScaled>(a.g[el.e], inv, c), a.eps1sq);
      a.p[el.e] = fmaf(step, u, __fmul_rn(a.p[el.e], decay));
      if (a.zero_grad) a.g[el.e] = 0.f;
    }
  }
}

template <bool kClip, bool kScaled>
int adafactor_launch_t(const AfArgs& a, cudaStream_t stream) {
  const unsigned blocks = (unsigned)(a.n_chunks < kAfMaxCtas ? a.n_chunks : kAfMaxCtas);
  const int smem = kAfSmemFloats * (int)sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(adafactor_stats_kernel<kClip, kScaled>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return (int)e;
  adafactor_stats_kernel<kClip, kScaled><<<blocks, kAfThreads, smem, stream>>>(a);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  adafactor_norm_kernel<kClip, kScaled><<<blocks, kAfThreads, 0, stream>>>(a);
  if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
  adafactor_apply_kernel<kClip, kScaled><<<blocks, kAfThreads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

}  // namespace b2

extern "C" {

// One FlatAdafactor update of a flat bucket on `stream`: the stats, norm and apply kernels.  max_norm > 0: g is clipped by
// the norm of grad_sqnorm's n_buckets sums.  cudaErrorInvalidValue, without a launch, for a null pointer, an empty or
// inconsistent table, a group count outside 1..kMaxGroups, or clipping without sqnorms.  The bindings check the table's rows.
int b2_adafactor_launch(const b2::AfArgs* a, cudaStream_t stream) {
  if (a == nullptr || a->p == nullptr || a->g == nullptr || a->state == nullptr || a->table == nullptr || a->partials == nullptr ||
      a->rc == nullptr || a->means == nullptr || a->tickets == nullptr || a->alpha == nullptr || a->step == nullptr)
    return (int)cudaErrorInvalidValue;
  if (a->n_tensors < 1 || a->n_chunks < 1 || (size_t)a->n_chunks > a->n || a->n_groups < 1 || a->n_groups > b2::kMaxGroups)
    return (int)cudaErrorInvalidValue;
  const bool clip = a->max_norm > 0.f;
  if (clip && (a->sqnorms == nullptr || a->n_buckets < 1 || !(a->max_norm < INFINITY))) return (int)cudaErrorInvalidValue;
  using namespace b2;
  switch ((clip ? 2 : 0) | (a->grad_scale != nullptr ? 1 : 0)) {
    case 0: return adafactor_launch_t<false, false>(*a, stream);
    case 1: return adafactor_launch_t<false, true>(*a, stream);
    case 2: return adafactor_launch_t<true, false>(*a, stream);
    default: return adafactor_launch_t<true, true>(*a, stream);
  }
}

}  // extern "C"
