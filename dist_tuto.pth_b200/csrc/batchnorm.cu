// SyncBatchNorm kernels (parallel/sync_bn.py): per-channel batch statistics in fp64, exchanged between the ranks by the
// existing fp64 SUM all-reduce, and the element-wise passes from coefficients rounded once to fp32.
//
// The input is seen in one of two layouts:
//   channels-last  [M rows, C]        (NHWC / NDHWC, or any [N, C] input): a CTA covers a tile of cx channel vectors of V
//                                      channels and a split of the rows; the 512 threads are 512/cx rows x cx lanes;
//   channel-first  [N, C, L]          (plain contiguous, L > 1): a CTA covers one channel (grid-strided) and a split of the
//                                      N x L/V vectors of that channel.
// V is 16 bytes of elements when the channel count (channels-last) or L (channel-first) and every pointer allow it, else 1.
//
// Reductions: every thread accumulates its elements in fp64 in a fixed order, a CTA adds its threads in a fixed tree
// (warp butterfly, then the warps in order), writes one partial per channel and split, and the last CTA of a tile to arrive
// (ticket per tile, reset by that CTA) adds the splits in split order.  The grid depends on the shape and max_blocks only, so
// a call is bit-reproducible run to run.  None of these kernels waits on a peer.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "batchnorm.h"

namespace b2 {
namespace bn {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kUnroll = 4;              // independent 16-byte loads in flight per thread
constexpr int kMaxTileCh = 32 * 8;      // channels of one channels-last tile (32 lanes x 8 bf16)


__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

template <typename T, int V>
__device__ __forceinline__ void load_vec(const T* __restrict__ p, float (&f)[V]) {
  if constexpr (V == 1) {
    f[0] = to_f(__ldg(p));
  } else {
    static_assert(V * sizeof(T) == 16, "a vector is 16 bytes");
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
    const T* e = reinterpret_cast<const T*>(&u);
#pragma unroll
    for (int k = 0; k < V; ++k) f[k] = to_f(e[k]);
  }
}

template <typename T, int V>
__device__ __forceinline__ void store_vec(T* p, const float (&f)[V]) {
  if constexpr (V == 1) {
    *p = from_f<T>(f[0]);
  } else {
    uint4 u;
    T* e = reinterpret_cast<T*>(&u);
#pragma unroll
    for (int k = 0; k < V; ++k) e[k] = from_f<T>(f[k]);
    *reinterpret_cast<uint4*>(p) = u;
  }
}

__device__ __forceinline__ double ld_param(const void* p, int code, int c) {
  if (code == 1) return (double)__bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[c]);
  if (code == 2) return (double)__half2float(reinterpret_cast<const __half*>(p)[c]);
  return (double)reinterpret_cast<const float*>(p)[c];
}
__device__ __forceinline__ void st_param(void* p, int code, int c, double v) {
  if (code == 1) reinterpret_cast<__nv_bfloat16*>(p)[c] = __double2bfloat16(v);
  else if (code == 2) reinterpret_cast<__half*>(p)[c] = __double2half(v);
  else reinterpret_cast<float*>(p)[c] = (float)v;
}

// Adds the CTA's per-thread pairs (s1[k], s2[k]) of channel lane (threadIdx % cx) in a fixed order and stores the CTA's
// partial of channel chan(lane, k) for split blockIdx.y; then the last CTA of the tile adds the splits in order and calls
// fin(c, q1, q2) for every channel of the tile.  Every thread of the CTA calls it.
template <int V, typename Chan, typename Fin>
__device__ __forceinline__ void reduce_tile(const Args& a, int tile, int cx, int tile_ch0, int tile_nch, double (&s1)[V],
                                            double (&s2)[V], Chan chan, Fin fin) {
  __shared__ double sm[kWarps][32][2];
  __shared__ int s_last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < V; ++k) {
    double p1 = s1[k], p2 = s2[k];
    for (int off = cx; off < 32; off <<= 1) {
      p1 += __shfl_xor_sync(0xffffffffu, p1, off);
      p2 += __shfl_xor_sync(0xffffffffu, p2, off);
    }
    if (lane < cx) { sm[warp][lane][0] = p1; sm[warp][lane][1] = p2; }
    __syncthreads();
    if ((int)threadIdx.x < cx) {
      double q1 = 0.0, q2 = 0.0;
      for (int w = 0; w < kWarps; ++w) { q1 += sm[w][threadIdx.x][0]; q2 += sm[w][threadIdx.x][1]; }
      const int c = chan(threadIdx.x, k);
      if (c >= 0) {
        __stcg(a.part + ((size_t)blockIdx.y * 2) * a.C + c, q1);
        __stcg(a.part + ((size_t)blockIdx.y * 2 + 1) * a.C + c, q2);
      }
    }
    __syncthreads();
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    s_last = atomicAdd(a.tickets + tile, 1u) == gridDim.y - 1;
    if (s_last) __threadfence();
  }
  __syncthreads();
  if (s_last) {
    for (int j = threadIdx.x; j < tile_nch; j += kThreads) {
      const int c = tile_ch0 + j;
      double q1 = 0.0, q2 = 0.0;
      for (int s = 0; s < (int)gridDim.y; ++s) {
        q1 += __ldcg(a.part + ((size_t)s * 2) * a.C + c);
        q2 += __ldcg(a.part + ((size_t)s * 2 + 1) * a.C + c);
      }
      fin(c, q1, q2);
    }
    if (threadIdx.x == 0) a.tickets[tile] = 0u;
  }
  __syncthreads();
}

// --------------------------------------------------------------------------------------------- forward statistics
// ex <- [local count | S1 = sum x (C) | S2 = sum x^2 (C) | zeros up to n_ex]
__device__ __forceinline__ void stats_fin(const Args& a, int c, double q1, double q2) {
  a.ex[1 + c] = q1;
  a.ex[1 + a.C + c] = q2;
}
__device__ __forceinline__ void stats_head(const Args& a) {
  if (blockIdx.x == 0 && blockIdx.y == 0) {
    if (threadIdx.x == 0) a.ex[0] = (double)a.count;
    for (int j = 1 + 2 * a.C + threadIdx.x; j < a.n_ex; j += kThreads) a.ex[j] = 0.0;
  }
}

template <typename T, int V>
__global__ void __launch_bounds__(kThreads, 1) bn_stats_cl_kernel(Args a) {
  stats_head(a);
  const int cx = a.cx, tx = threadIdx.x % cx, ry = threadIdx.x / cx, rt = kThreads / cx;
  const long long r0 = (long long)blockIdx.y * a.per_split, r1 = min(a.rows, r0 + a.per_split);
  for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
    const int cvi = tile * cx + tx;
    double s1[V], s2[V];
#pragma unroll
    for (int k = 0; k < V; ++k) s1[k] = s2[k] = 0.0;
    if (cvi < a.cv) {
      const T* x = reinterpret_cast<const T*>(a.x) + (size_t)cvi * V;
      long long r = r0 + ry;
      for (; r + (kUnroll - 1) * rt < r1; r += kUnroll * rt) {
        float f[kUnroll][V];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) load_vec<T, V>(x + (size_t)(r + u * rt) * a.C, f[u]);
#pragma unroll
        for (int u = 0; u < kUnroll; ++u)
#pragma unroll
          for (int k = 0; k < V; ++k) { const double d = f[u][k]; s1[k] += d; s2[k] = fma(d, d, s2[k]); }
      }
      for (; r < r1; r += rt) {
        float f[V];
        load_vec<T, V>(x + (size_t)r * a.C, f);
#pragma unroll
        for (int k = 0; k < V; ++k) { const double d = f[k]; s1[k] += d; s2[k] = fma(d, d, s2[k]); }
      }
    }
    const int ch0 = tile * cx * V;
    reduce_tile<V>(a, tile, cx, ch0, min(cx * V, a.C - ch0), s1, s2,
                   [&](int l, int k) { const int v = tile * cx + l; return v < a.cv ? v * V + k : -1; },
                   [&](int c, double q1, double q2) { stats_fin(a, c, q1, q2); });
  }
}

// channel-first: vector j of channel c is element ((n * C + c) * L + lv * V), n = j / Lv
template <typename T, int V>
__device__ __forceinline__ const T* cf_ptr(const Args& a, const void* base, int c, long long j) {
  const long long n = j / a.Lv, lv = j - n * a.Lv;
  return reinterpret_cast<const T*>(base) + ((size_t)n * a.C + c) * (size_t)(a.Lv * V) + (size_t)lv * V;
}

template <typename T, int V>
__global__ void __launch_bounds__(kThreads, 1) bn_stats_cf_kernel(Args a) {
  stats_head(a);
  const long long j0 = (long long)blockIdx.y * a.per_split, j1 = min(a.rows, j0 + a.per_split);
  for (int c = blockIdx.x; c < a.C; c += gridDim.x) {
    double s1[1] = {0.0}, s2[1] = {0.0};
    long long j = j0 + threadIdx.x;
    for (; j + (kUnroll - 1) * kThreads < j1; j += kUnroll * kThreads) {
      float f[kUnroll][V];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) load_vec<T, V>(cf_ptr<T, V>(a, a.x, c, j + u * kThreads), f[u]);
#pragma unroll
      for (int u = 0; u < kUnroll; ++u)
#pragma unroll
        for (int k = 0; k < V; ++k) { const double d = f[u][k]; s1[0] += d; s2[0] = fma(d, d, s2[0]); }
    }
    for (; j < j1; j += kThreads) {
      float f[V];
      load_vec<T, V>(cf_ptr<T, V>(a, a.x, c, j), f);
#pragma unroll
      for (int k = 0; k < V; ++k) { const double d = f[k]; s1[0] += d; s2[0] = fma(d, d, s2[0]); }
    }
    reduce_tile<1>(a, c, 1, c, 1, s1, s2, [&](int, int) { return c; },
                   [&](int cc, double q1, double q2) { stats_fin(a, cc, q1, q2); });
  }
}

// --------------------------------------------------------------------------------------------- forward apply
// From the exchanged sums: mean = S1/N, var = max(S2/N - mean^2, 0), invstd = 1/sqrt(var + eps) (fp64); k1 = w invstd and
// k0 = b - mean k1 rounded once to fp32.  `owner`: this CTA also saves mean / invstd / N and updates the running stats.
__device__ __forceinline__ void coef_fwd(const Args& a, int c, bool owner, float& k1, float& k0) {
  const double N = a.ex[0];
  const double mean = a.ex[1 + c] / N;
  const double var = fmax(a.ex[1 + a.C + c] / N - mean * mean, 0.0);
  const double invstd = 1.0 / sqrt(var + a.eps);
  const double w = a.w ? ld_param(a.w, a.pw, c) : 1.0, b = a.b ? ld_param(a.b, a.pw, c) : 0.0;
  const double d1 = w * invstd;
  k1 = (float)d1;
  k0 = (float)(b - mean * d1);
  if (!owner) return;
  a.stats[c] = mean;
  a.stats[a.C + c] = invstd;
  if (c == 0) a.stats[2 * a.C] = N;
  if (a.rmean) {
    const double m = a.nbt ? 1.0 / (double)*a.nbt : a.momentum;
    st_param(a.rmean, a.pr, c, (1.0 - m) * ld_param(a.rmean, a.pr, c) + m * mean);
    st_param(a.rvar, a.pr, c, (1.0 - m) * ld_param(a.rvar, a.pr, c) + m * (var * N / (N - 1.0)));
  }
}

template <typename T, int V>
__global__ void __launch_bounds__(kThreads, 1) bn_apply_cl_kernel(Args a) {
  __shared__ float sk1[kMaxTileCh], sk0[kMaxTileCh];
  const int cx = a.cx, tx = threadIdx.x % cx, ry = threadIdx.x / cx, rt = kThreads / cx;
  const long long r0 = (long long)blockIdx.y * a.per_split, r1 = min(a.rows, r0 + a.per_split);
  for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
    const int ch0 = tile * cx * V, nch = min(cx * V, a.C - ch0);
    for (int j = threadIdx.x; j < nch; j += kThreads) coef_fwd(a, ch0 + j, blockIdx.y == 0, sk1[j], sk0[j]);
    __syncthreads();
    const int cvi = tile * cx + tx;
    if (cvi < a.cv) {
      float k1[V], k0[V];
#pragma unroll
      for (int k = 0; k < V; ++k) { k1[k] = sk1[tx * V + k]; k0[k] = sk0[tx * V + k]; }
      const T* x = reinterpret_cast<const T*>(a.x) + (size_t)cvi * V;
      T* y = reinterpret_cast<T*>(a.y) + (size_t)cvi * V;
      long long r = r0 + ry;
      for (; r + (kUnroll - 1) * rt < r1; r += kUnroll * rt) {
        float f[kUnroll][V];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) load_vec<T, V>(x + (size_t)(r + u * rt) * a.C, f[u]);
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
#pragma unroll
          for (int k = 0; k < V; ++k) f[u][k] = fmaf(f[u][k], k1[k], k0[k]);
          store_vec<T, V>(y + (size_t)(r + u * rt) * a.C, f[u]);
        }
      }
      for (; r < r1; r += rt) {
        float f[V];
        load_vec<T, V>(x + (size_t)r * a.C, f);
#pragma unroll
        for (int k = 0; k < V; ++k) f[k] = fmaf(f[k], k1[k], k0[k]);
        store_vec<T, V>(y + (size_t)r * a.C, f);
      }
    }
    __syncthreads();
  }
}

template <typename T, int V>
__global__ void __launch_bounds__(kThreads, 1) bn_apply_cf_kernel(Args a) {
  __shared__ float sk[2];
  const long long j0 = (long long)blockIdx.y * a.per_split, j1 = min(a.rows, j0 + a.per_split);
  for (int c = blockIdx.x; c < a.C; c += gridDim.x) {
    if (threadIdx.x == 0) coef_fwd(a, c, blockIdx.y == 0, sk[0], sk[1]);
    __syncthreads();
    const float k1 = sk[0], k0 = sk[1];
    for (long long j = j0 + threadIdx.x; j < j1; j += kThreads) {
      float f[V];
      const T* xp = cf_ptr<T, V>(a, a.x, c, j);
      load_vec<T, V>(xp, f);
#pragma unroll
      for (int k = 0; k < V; ++k) f[k] = fmaf(f[k], k1, k0);
      store_vec<T, V>(reinterpret_cast<T*>(a.y) + (xp - reinterpret_cast<const T*>(a.x)), f);
    }
    __syncthreads();
  }
}

// --------------------------------------------------------------------------------------------- backward reduce
// ex <- [sum dy (C) | sum dy (x - mean) (C) | zeros up to n_ex] (local); grad_bias = sum dy, grad_weight = sum dy xmu invstd.
__device__ __forceinline__ void bwd_fin(const Args& a, int c, double q1, double q2) {
  a.ex[c] = q1;
  a.ex[a.C + c] = q2;
  if (a.gb) st_param(a.gb, a.pw, c, q1);
  if (a.gw) st_param(a.gw, a.pw, c, q2 * a.stats[a.C + c]);
}
__device__ __forceinline__ void bwd_head(const Args& a) {
  if (blockIdx.x == 0 && blockIdx.y == 0)
    for (int j = 2 * a.C + threadIdx.x; j < a.n_ex; j += kThreads) a.ex[j] = 0.0;
}

template <typename T, int V>
__global__ void __launch_bounds__(kThreads, 1) bn_backward_reduce_cl_kernel(Args a) {
  bwd_head(a);
  const int cx = a.cx, tx = threadIdx.x % cx, ry = threadIdx.x / cx, rt = kThreads / cx;
  const long long r0 = (long long)blockIdx.y * a.per_split, r1 = min(a.rows, r0 + a.per_split);
  for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
    const int cvi = tile * cx + tx;
    double s1[V], s2[V];
#pragma unroll
    for (int k = 0; k < V; ++k) s1[k] = s2[k] = 0.0;
    if (cvi < a.cv) {
      double mean[V];
#pragma unroll
      for (int k = 0; k < V; ++k) mean[k] = a.stats[cvi * V + k];
      const T* x = reinterpret_cast<const T*>(a.x) + (size_t)cvi * V;
      const T* dy = reinterpret_cast<const T*>(a.dy) + (size_t)cvi * V;
      long long r = r0 + ry;
      for (; r + (kUnroll / 2 - 1) * rt < r1; r += (kUnroll / 2) * rt) {
        float f[kUnroll / 2][V], g[kUnroll / 2][V];
#pragma unroll
        for (int u = 0; u < kUnroll / 2; ++u) {
          load_vec<T, V>(x + (size_t)(r + u * rt) * a.C, f[u]);
          load_vec<T, V>(dy + (size_t)(r + u * rt) * a.C, g[u]);
        }
#pragma unroll
        for (int u = 0; u < kUnroll / 2; ++u)
#pragma unroll
          for (int k = 0; k < V; ++k) {
            const double d = g[u][k];
            s1[k] += d;
            s2[k] = fma(d, (double)f[u][k] - mean[k], s2[k]);
          }
      }
      for (; r < r1; r += rt) {
        float f[V], g[V];
        load_vec<T, V>(x + (size_t)r * a.C, f);
        load_vec<T, V>(dy + (size_t)r * a.C, g);
#pragma unroll
        for (int k = 0; k < V; ++k) { const double d = g[k]; s1[k] += d; s2[k] = fma(d, (double)f[k] - mean[k], s2[k]); }
      }
    }
    const int ch0 = tile * cx * V;
    reduce_tile<V>(a, tile, cx, ch0, min(cx * V, a.C - ch0), s1, s2,
                   [&](int l, int k) { const int v = tile * cx + l; return v < a.cv ? v * V + k : -1; },
                   [&](int c, double q1, double q2) { bwd_fin(a, c, q1, q2); });
  }
}

template <typename T, int V>
__global__ void __launch_bounds__(kThreads, 1) bn_backward_reduce_cf_kernel(Args a) {
  bwd_head(a);
  const long long j0 = (long long)blockIdx.y * a.per_split, j1 = min(a.rows, j0 + a.per_split);
  for (int c = blockIdx.x; c < a.C; c += gridDim.x) {
    const double mean = a.stats[c];
    double s1[1] = {0.0}, s2[1] = {0.0};
    long long j = j0 + threadIdx.x;
    for (; j + (kUnroll / 2 - 1) * kThreads < j1; j += (kUnroll / 2) * kThreads) {
      float f[kUnroll / 2][V], g[kUnroll / 2][V];
#pragma unroll
      for (int u = 0; u < kUnroll / 2; ++u) {
        load_vec<T, V>(cf_ptr<T, V>(a, a.x, c, j + u * kThreads), f[u]);
        load_vec<T, V>(cf_ptr<T, V>(a, a.dy, c, j + u * kThreads), g[u]);
      }
#pragma unroll
      for (int u = 0; u < kUnroll / 2; ++u)
#pragma unroll
        for (int k = 0; k < V; ++k) { const double d = g[u][k]; s1[0] += d; s2[0] = fma(d, (double)f[u][k] - mean, s2[0]); }
    }
    for (; j < j1; j += kThreads) {
      float f[V], g[V];
      load_vec<T, V>(cf_ptr<T, V>(a, a.x, c, j), f);
      load_vec<T, V>(cf_ptr<T, V>(a, a.dy, c, j), g);
#pragma unroll
      for (int k = 0; k < V; ++k) { const double d = g[k]; s1[0] += d; s2[0] = fma(d, (double)f[k] - mean, s2[0]); }
    }
    reduce_tile<1>(a, c, 1, c, 1, s1, s2, [&](int, int) { return c; },
                   [&](int cc, double q1, double q2) { bwd_fin(a, cc, q1, q2); });
  }
}

// --------------------------------------------------------------------------------------------- backward apply
// dx = w invstd (dy - Sdy/N - (x - mean) invstd^2 Sdyxmu/N) = dy ka + x kb + kc, the coefficients from fp64 rounded once.
__device__ __forceinline__ void coef_bwd(const Args& a, int c, float& ka, float& kb, float& kc) {
  const double N = a.stats[2 * a.C], mean = a.stats[c], invstd = a.stats[a.C + c];
  const double w = a.w ? ld_param(a.w, a.pw, c) : 1.0;
  const double da = w * invstd;
  const double db = -da * invstd * invstd * (a.ex[a.C + c] / N);
  ka = (float)da;
  kb = (float)db;
  kc = (float)(-da * (a.ex[c] / N) - db * mean);
}

template <typename T, int V>
__global__ void __launch_bounds__(kThreads, 1) bn_backward_apply_cl_kernel(Args a) {
  __shared__ float ska[kMaxTileCh], skb[kMaxTileCh], skc[kMaxTileCh];
  const int cx = a.cx, tx = threadIdx.x % cx, ry = threadIdx.x / cx, rt = kThreads / cx;
  const long long r0 = (long long)blockIdx.y * a.per_split, r1 = min(a.rows, r0 + a.per_split);
  for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
    const int ch0 = tile * cx * V, nch = min(cx * V, a.C - ch0);
    for (int j = threadIdx.x; j < nch; j += kThreads) coef_bwd(a, ch0 + j, ska[j], skb[j], skc[j]);
    __syncthreads();
    const int cvi = tile * cx + tx;
    if (cvi < a.cv) {
      float ka[V], kb[V], kc[V];
#pragma unroll
      for (int k = 0; k < V; ++k) { ka[k] = ska[tx * V + k]; kb[k] = skb[tx * V + k]; kc[k] = skc[tx * V + k]; }
      const size_t off = (size_t)cvi * V;
      const T* x = reinterpret_cast<const T*>(a.x) + off;
      const T* dy = reinterpret_cast<const T*>(a.dy) + off;
      T* dx = reinterpret_cast<T*>(a.dx) + off;
      for (long long r = r0 + ry; r < r1; r += rt) {
        float f[V], g[V];
        load_vec<T, V>(x + (size_t)r * a.C, f);
        load_vec<T, V>(dy + (size_t)r * a.C, g);
#pragma unroll
        for (int k = 0; k < V; ++k) g[k] = fmaf(g[k], ka[k], fmaf(f[k], kb[k], kc[k]));
        store_vec<T, V>(dx + (size_t)r * a.C, g);
      }
    }
    __syncthreads();
  }
}

template <typename T, int V>
__global__ void __launch_bounds__(kThreads, 1) bn_backward_apply_cf_kernel(Args a) {
  __shared__ float sk[3];
  const long long j0 = (long long)blockIdx.y * a.per_split, j1 = min(a.rows, j0 + a.per_split);
  for (int c = blockIdx.x; c < a.C; c += gridDim.x) {
    if (threadIdx.x == 0) coef_bwd(a, c, sk[0], sk[1], sk[2]);
    __syncthreads();
    const float ka = sk[0], kb = sk[1], kc = sk[2];
    for (long long j = j0 + threadIdx.x; j < j1; j += kThreads) {
      float f[V], g[V];
      const T* xp = cf_ptr<T, V>(a, a.x, c, j);
      const size_t e = xp - reinterpret_cast<const T*>(a.x);
      load_vec<T, V>(xp, f);
      load_vec<T, V>(reinterpret_cast<const T*>(a.dy) + e, g);
#pragma unroll
      for (int k = 0; k < V; ++k) g[k] = fmaf(g[k], ka, fmaf(f[k], kb, kc));
      store_vec<T, V>(reinterpret_cast<T*>(a.dx) + e, g);
    }
    __syncthreads();
  }
}

// --------------------------------------------------------------------------------------------- launch
// Geometry from the shape and max_blocks: the grid never exceeds max_blocks CTAs; a split holds at least kUnroll rows
// (vectors) per thread, so small tensors take few CTAs.
inline void geometry(Args& a, bool cl, int V, long long M, long long L, int max_blocks, dim3& grid) {
  if (max_blocks < 1) max_blocks = 1;
  const long long vec_per_split_min = (long long)kThreads * kUnroll;
  if (cl) {
    a.cv = (a.C + V - 1) / V;
    int cx = 1;
    while (cx < a.cv && cx < 32) cx <<= 1;
    a.cx = cx;
    a.tiles = (a.cv + cx - 1) / cx;
    a.rows = M;
    a.Lv = 1;
    const int gx = a.tiles < max_blocks ? a.tiles : max_blocks;
    long long gy = max_blocks / gx;
    const long long by_size = (M * cx + vec_per_split_min - 1) / vec_per_split_min;
    if (gy > by_size) gy = by_size;
    if (gy < 1) gy = 1;
    a.per_split = (M + gy - 1) / gy;
    grid = dim3((unsigned)gx, (unsigned)gy);
  } else {
    a.cv = a.C;
    a.cx = 1;
    a.tiles = a.C;
    a.Lv = L / V;
    a.rows = M * a.Lv;
    const int gx = a.C < max_blocks ? a.C : max_blocks;
    long long gy = max_blocks / gx;
    const long long by_size = (a.rows + vec_per_split_min - 1) / vec_per_split_min;
    if (gy > by_size) gy = by_size;
    if (gy < 1) gy = 1;
    a.per_split = (a.rows + gy - 1) / gy;
    grid = dim3((unsigned)gx, (unsigned)gy);
  }
  if (a.per_split < 1) a.per_split = 1;
}

#define B2_BN_DISPATCH(NAME)                                                                                        \
  template <typename T, int V>                                                                                      \
  struct NAME##_k {                                                                                                 \
    static void launch(bool cl, dim3 g, const Args& a, cudaStream_t s) {                                            \
      if (cl) NAME##_cl_kernel<T, V><<<g, kThreads, 0, s>>>(a);                                                     \
      else NAME##_cf_kernel<T, V><<<g, kThreads, 0, s>>>(a);                                                        \
    }                                                                                                               \
  };
B2_BN_DISPATCH(bn_stats)
B2_BN_DISPATCH(bn_apply)
B2_BN_DISPATCH(bn_backward_reduce)
B2_BN_DISPATCH(bn_backward_apply)
#undef B2_BN_DISPATCH

template <template <typename, int> class K>
int launch(int dtype, int vec, bool cl, long long M, long long L, int max_blocks, Args a, dim3* grid_out, cudaStream_t s) {
  const int V = vec ? (dtype == 0 ? 4 : 8) : 1;
  dim3 grid;
  geometry(a, cl, V, M, L, max_blocks, grid);
  if (grid_out) { *grid_out = grid; return 0; }
  if (dtype == 0) { if (vec) K<float, 4>::launch(cl, grid, a, s); else K<float, 1>::launch(cl, grid, a, s); }
  else if (dtype == 1) { if (vec) K<__nv_bfloat16, 8>::launch(cl, grid, a, s); else K<__nv_bfloat16, 1>::launch(cl, grid, a, s); }
  else { if (vec) K<__half, 8>::launch(cl, grid, a, s); else K<__half, 1>::launch(cl, grid, a, s); }
  return (int)cudaGetLastError();
}

}  // namespace bn
}  // namespace b2

extern "C" {

// kind: 0 forward statistics, 1 forward apply, 2 backward reduce, 3 backward apply.  dtype: 0 fp32, 1 bf16, 2 fp16 (input).
// vec: 16-byte vectors (the caller checked divisibility and alignment).  cl: channels-last [M, C]; else [M, C, L].
// With grid_out set nothing is launched: the grid the call would use (its y extent sizes the partials) is returned.
int b2_bn_launch(int kind, int dtype, int vec, int cl, long long M, long long L, int max_blocks, const b2::bn::Args* args,
                 unsigned int* grid_out, cudaStream_t stream) {
  dim3 g;
  dim3* gp = grid_out ? &g : nullptr;
  int rc;
  switch (kind) {
    case 0: rc = b2::bn::launch<b2::bn::bn_stats_k>(dtype, vec, cl, M, L, max_blocks, *args, gp, stream); break;
    case 1: rc = b2::bn::launch<b2::bn::bn_apply_k>(dtype, vec, cl, M, L, max_blocks, *args, gp, stream); break;
    case 2: rc = b2::bn::launch<b2::bn::bn_backward_reduce_k>(dtype, vec, cl, M, L, max_blocks, *args, gp, stream); break;
    default: rc = b2::bn::launch<b2::bn::bn_backward_apply_k>(dtype, vec, cl, M, L, max_blocks, *args, gp, stream); break;
  }
  if (grid_out) { grid_out[0] = g.x; grid_out[1] = g.y; }
  return rc;
}

size_t b2_bn_args_size() { return sizeof(b2::bn::Args); }

}  // extern "C"
