// FlatLAMB's and FlatLARS's sharded update of one gradient bucket on sm_90a (ops/optim.py, sharded=True on one peer-memory
// world): ZeRO stage 1 for the layer-wise optimizers.  It runs where the all-reduce would have run, in two launches per bucket
// on every rank, with the same grid on every rank (shard_grid.h; the per-block barriers pair block b of every rank).
//
// Rank r owns the elements [lo, lo + per) of the padded bucket (lo = r * per), keeps the optimizer state of that slice only,
// and has its own chunk table (layerwise.h): each tensor's piece of the slice cut into chunks of at most kLwChunk elements from
// the piece's start, so no chunk crosses a tensor or a slice boundary; the tensor rows are those of all T tensors of the
// bucket (a tensor without a piece in the slice has no chunk here).
//
//   sharded_layerwise_norms_kernel   barrier: every rank's gradients of this bucket are complete.  Per chunk of this rank's
//                                    table: g = (((0 + g_0) + g_1) + ...) * scale in fp32 in rank order (what sharded_step_kernel
//                                    and the all-reduce form, fp32 or bf16 buckets); LAMB updates the m / v shards and forms u,
//                                    LARS keeps g in a workspace shard; both sum p^2 and u^2 (LAMB) or g^2 (LARS) in
//                                    layerwise_norms_kernel's order, and the last CTA of a tensor adds its chunk partials in
//                                    chunk order in fp64 into this rank's sums[2t], sums[2t + 1] (0 for a tensor without a piece
//                                    here).  The gradients are not zeroed: the peers are still reading them.
//   sharded_layerwise_apply_kernel   barrier: every rank finished the norms kernel, so every rank's sums are complete and no
//                                    peer reads this rank's gradients any more.  A tensor's two sums are the W ranks' sums added
//                                    in rank order from +0 in fp64 (read from the peers' symmetric sums buffers: the same bits on
//                                    every rank), and its ratio is layerwise_apply_kernel's.  Every rank writes the ratios of
//                                    all T tensors.  The update of the owned slice (LAMB: u recomputed from the stored moments;
//                                    LARS: lars_elem on the kept gradient) is stored into EVERY rank's parameter flat.  Barrier:
//                                    every slice has landed everywhere; then the local bucket is zeroed (zero_grad).
//
// NVLink traffic is sharded_step_kernel's: every gradient slice is read once from every peer (norms kernel) and every parameter
// slice stored once to every peer (apply kernel), plus the per-tensor sums: each chunk's CTA reads its tensor's 16 bytes from
// every rank, and the ratio pass reads 16 bytes per tensor from every rank.
#include <cstring>
#include "common.cuh"
#include "layerwise_device.cuh"
#include "shard_grid.h"

namespace b2 {

struct ShardedLwArgs {
  PeerPtrs grads;         // every rank's gradient bucket: n_vec 16-byte vectors (4 fp32 or 8 bf16 gradients each)
  PeerPtrs params;        // every rank's fp32 parameter flat
  PeerPtrs sums;          // every rank's fp64 [2 * n_tensors]: the sums over that rank's chunks
  SignalPads sig;         // signal pad of the gradient bucket
  // this rank's table, partials, tickets, ratios and scalars.  p: its own parameter flat, sums: its own sums buffer, m / v:
  // its state shards and g (LARS) its averaged-gradient workspace, all indexed from the slice start; n: slice elements.
  LwArgs lw;
  size_t n_vec, lo;       // lo: the slice's first element in the bucket
  float scale;
  int rank, world;
};

// g = (((0 + g_0) + g_1) + ...) * scale in fp32, rank order, at the 4 elements from e (a multiple of 4); every rank's vector
// is loaded before the first add
template <bool kBf16>
__device__ __forceinline__ float4 rank_sum4(const ShardedLwArgs& a, size_t e) {
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
  if constexpr (kBf16) {
    uint2 raw[B2_MAX_RANKS];
#pragma unroll
    for (int r = 0; r < B2_MAX_RANKS; ++r)
      if (r < a.world) raw[r] = __ldcg(reinterpret_cast<const uint2*>(a.grads.p[r]) + e / 4);
#pragma unroll
    for (int r = 0; r < B2_MAX_RANKS; ++r) {
      if (r < a.world) {
        g.x = __fadd_rn(g.x, bf16lo(raw[r].x)); g.y = __fadd_rn(g.y, bf16hi(raw[r].x));
        g.z = __fadd_rn(g.z, bf16lo(raw[r].y)); g.w = __fadd_rn(g.w, bf16hi(raw[r].y));
      }
    }
  } else {
    uint4 raw[B2_MAX_RANKS];
#pragma unroll
    for (int r = 0; r < B2_MAX_RANKS; ++r)
      if (r < a.world) raw[r] = ld_cg_v4(reinterpret_cast<const uint4*>(a.grads.p[r]) + e / 4);
#pragma unroll
    for (int r = 0; r < B2_MAX_RANKS; ++r) {
      if (r < a.world) {
        g.x = __fadd_rn(g.x, __uint_as_float(raw[r].x)); g.y = __fadd_rn(g.y, __uint_as_float(raw[r].y));
        g.z = __fadd_rn(g.z, __uint_as_float(raw[r].z)); g.w = __fadd_rn(g.w, __uint_as_float(raw[r].w));
      }
    }
  }
  return make_float4(__fmul_rn(g.x, a.scale), __fmul_rn(g.y, a.scale), __fmul_rn(g.z, a.scale), __fmul_rn(g.w, a.scale));
}

// The same for the one element e (a tensor's tail)
template <bool kBf16>
__device__ __forceinline__ float rank_sum1(const ShardedLwArgs& a, size_t e) {
  float g = 0.f;
  for (int r = 0; r < a.world; ++r) {
    const float x = kBf16 ? __uint_as_float((uint32_t)__ldcg(reinterpret_cast<const unsigned short*>(a.grads.p[r]) + e) << 16)
                          : __ldcg(reinterpret_cast<const float*>(a.grads.p[r]) + e);
    g = __fadd_rn(g, x);
  }
  return __fmul_rn(g, a.scale);
}

template <bool kBf16, bool kLamb>
__global__ void __launch_bounds__(kLwThreads) sharded_layerwise_norms_kernel(const ShardedLwArgs sa) {
  __shared__ float2 s_warp[kLwThreads / 32];
  __shared__ float2 s_stage[kLwThreads];
  __shared__ int s_last;
  const LwArgs& a = sa.lw;
  uint32_t epoch = barrier_epoch_load(sa.sig, sa.rank);
  block_barrier_all_ranks(sa.sig, sa.rank, sa.world, ++epoch);       // every rank's gradients of this bucket are complete
  const long long* chunks = a.table;
  const long long* tens = a.table + (size_t)a.n_chunks * kLwRow;
  for (int t = blockIdx.x * kLwThreads + threadIdx.x; t < a.n_tensors; t += gridDim.x * kLwThreads) {
    if (tens[t * kLwRow + 1] == 0) {          // no piece in this slice: it adds 0 to the exchange
      a.sums[2 * t] = 0.0;
      a.sums[2 * t + 1] = 0.0;
    }
  }
  for (int ch = blockIdx.x; ch < a.n_chunks; ch += gridDim.x) {
    const long long start = chunks[ch * kLwRow], len = chunks[ch * kLwRow + 1];
    const int t = (int)chunks[ch * kLwRow + 2];
    const float wd = kLamb && tens[t * kLwRow + 2] != 0 ? a.wd : 0.f;
    const int nv = (int)(len >> 2), tail = (int)(len & 3);
    const size_t v0 = (size_t)start >> 2;                   // bucket coordinates: p and the gradient buckets
    const size_t q0 = (size_t)(start - (long long)sa.lo) >> 2;   // slice coordinates: the state shards and the workspace
    float sp = 0.f, sq = 0.f;
    for (int i = threadIdx.x; i < nv; i += kLwThreads) {
      const float4 gv = rank_sum4<kBf16>(sa, (v0 + i) * 4);
      const float4 pv = reinterpret_cast<const float4*>(a.p)[v0 + i];
      sp = fmaf(pv.x, pv.x, sp); sp = fmaf(pv.y, pv.y, sp); sp = fmaf(pv.z, pv.z, sp); sp = fmaf(pv.w, pv.w, sp);
      if constexpr (kLamb) {
        float4 mv = reinterpret_cast<const float4*>(a.m)[q0 + i];
        float4 vv = reinterpret_cast<const float4*>(a.v)[q0 + i];
        adam_moments(mv.x, vv.x, gv.x, a);
        adam_moments(mv.y, vv.y, gv.y, a);
        adam_moments(mv.z, vv.z, gv.z, a);
        adam_moments(mv.w, vv.w, gv.w, a);
        reinterpret_cast<float4*>(a.m)[q0 + i] = mv;
        reinterpret_cast<float4*>(a.v)[q0 + i] = vv;
        const float ux = lamb_u(pv.x, mv.x, vv.x, wd, a), uy = lamb_u(pv.y, mv.y, vv.y, wd, a);
        const float uz = lamb_u(pv.z, mv.z, vv.z, wd, a), uw = lamb_u(pv.w, mv.w, vv.w, wd, a);
        sq = fmaf(ux, ux, sq); sq = fmaf(uy, uy, sq); sq = fmaf(uz, uz, sq); sq = fmaf(uw, uw, sq);
      } else {
        reinterpret_cast<float4*>(a.g)[q0 + i] = gv;
        sq = fmaf(gv.x, gv.x, sq); sq = fmaf(gv.y, gv.y, sq); sq = fmaf(gv.z, gv.z, sq); sq = fmaf(gv.w, gv.w, sq);
      }
    }
    if (threadIdx.x < tail) {                  // a tensor's last < 4 elements: threads 0..2, one each
      const size_t e = (size_t)start + (size_t)nv * 4 + threadIdx.x, eq = e - sa.lo;
      const float pe = a.p[e];
      const float ge = rank_sum1<kBf16>(sa, e);
      sp = fmaf(pe, pe, sp);
      if constexpr (kLamb) {
        float me = a.m[eq], ve = a.v[eq];
        adam_moments(me, ve, ge, a);
        a.m[eq] = me;
        a.v[eq] = ve;
        const float u = lamb_u(pe, me, ve, wd, a);
        sq = fmaf(u, u, sq);
      } else {
        a.g[eq] = ge;
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
    if (s_last) {                              // uniform: the tensor's partials of this slice, in chunk order, in fp64
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
  if (threadIdx.x == 0) barrier_epoch_store(sa.sig, sa.rank, epoch);
}

// Tensor t's ratio from the W ranks' sums added in rank order from +0 in fp64; the rest is layerwise_apply_kernel's formula
template <bool kLamb>
__device__ __forceinline__ float sharded_ratio(const ShardedLwArgs& sa, int t, bool adapt) {
  double sp = 0.0, sq = 0.0;
  for (int r = 0; r < sa.world; ++r) {
    const double* s = reinterpret_cast<const double*>(sa.sums.p[r]) + 2 * t;
    sp = __dadd_rn(sp, __ldcg(s));
    sq = __dadd_rn(sq, __ldcg(s + 1));
  }
  const LwArgs& a = sa.lw;
  const double w = __dsqrt_rn(sp), q = __dsqrt_rn(sq);
  float r = 1.f;
  if (adapt && w > 0.0 && q > 0.0)
    r = kLamb ? __double2float_rn(__ddiv_rn(w, q))
              : __double2float_rn(__ddiv_rn(__dmul_rn(a.eta64, w), __dadd_rn(__dadd_rn(q, __dmul_rn(a.wd64, w)), a.eps64)));
  return r;
}

__device__ __forceinline__ void store_all_ranks(const ShardedLwArgs& sa, size_t v, float4 p) {
  const uint4 u = make_uint4(__float_as_uint(p.x), __float_as_uint(p.y), __float_as_uint(p.z), __float_as_uint(p.w));
#pragma unroll
  for (int r = 0; r < B2_MAX_RANKS; ++r)
    if (r < sa.world) st_cg_v4(reinterpret_cast<uint4*>(sa.params.p[r]) + v, u);
}

__device__ __forceinline__ void store_all_ranks1(const ShardedLwArgs& sa, size_t e, float p) {
  for (int r = 0; r < sa.world; ++r) __stcg(reinterpret_cast<float*>(sa.params.p[r]) + e, p);
}

template <bool kLamb>
__global__ void __launch_bounds__(kLwThreads) sharded_layerwise_apply_kernel(const ShardedLwArgs sa) {
  __shared__ float s_r;
  const LwArgs& a = sa.lw;
  const int rank = sa.rank, world = sa.world;
  uint32_t epoch = barrier_epoch_load(sa.sig, rank);
  // every rank finished the norms kernel: its sums are complete, and no peer reads this rank's gradients any more
  block_barrier_all_ranks(sa.sig, rank, world, ++epoch);
  const long long* chunks = a.table;
  const long long* tens = a.table + (size_t)a.n_chunks * kLwRow;
  for (int t = blockIdx.x * kLwThreads + threadIdx.x; t < a.n_tensors; t += gridDim.x * kLwThreads)
    a.ratios[t] = sharded_ratio<kLamb>(sa, t, tens[t * kLwRow + 2] != 0);
  for (int ch = blockIdx.x; ch < a.n_chunks; ch += gridDim.x) {
    const long long start = chunks[ch * kLwRow], len = chunks[ch * kLwRow + 1];
    const int t = (int)chunks[ch * kLwRow + 2];
    const bool adapt = tens[t * kLwRow + 2] != 0;
    __syncthreads();                           // the previous chunk's readers of s_r are done
    if (threadIdx.x == 0) s_r = sharded_ratio<kLamb>(sa, t, adapt);
    __syncthreads();
    const float r = s_r;
    const float wd = adapt ? a.wd : 0.f;
    const int nv = (int)(len >> 2), tail = (int)(len & 3);
    const size_t v0 = (size_t)start >> 2;
    const size_t q0 = (size_t)(start - (long long)sa.lo) >> 2;
    if constexpr (kLamb) {
      const float step = -__fmul_rn(a.lr, r);
      for (int i = threadIdx.x; i < nv; i += kLwThreads) {
        float4 pv = reinterpret_cast<const float4*>(a.p)[v0 + i];
        const float4 mv = reinterpret_cast<const float4*>(a.m)[q0 + i];
        const float4 vv = reinterpret_cast<const float4*>(a.v)[q0 + i];
        pv.x = fmaf(step, lamb_u(pv.x, mv.x, vv.x, wd, a), pv.x);
        pv.y = fmaf(step, lamb_u(pv.y, mv.y, vv.y, wd, a), pv.y);
        pv.z = fmaf(step, lamb_u(pv.z, mv.z, vv.z, wd, a), pv.z);
        pv.w = fmaf(step, lamb_u(pv.w, mv.w, vv.w, wd, a), pv.w);
        store_all_ranks(sa, v0 + i, pv);
      }
      if (threadIdx.x < tail) {
        const size_t e = (size_t)start + (size_t)nv * 4 + threadIdx.x, eq = e - sa.lo;
        store_all_ranks1(sa, e, fmaf(step, lamb_u(a.p[e], a.m[eq], a.v[eq], wd, a), a.p[e]));
      }
    } else {
      for (int i = threadIdx.x; i < nv; i += kLwThreads) {
        float4 pv = reinterpret_cast<const float4*>(a.p)[v0 + i];
        float4 mv = reinterpret_cast<const float4*>(a.m)[q0 + i];
        const float4 gv = reinterpret_cast<const float4*>(a.g)[q0 + i];
        lars_elem(pv.x, mv.x, gv.x, r, wd, a);
        lars_elem(pv.y, mv.y, gv.y, r, wd, a);
        lars_elem(pv.z, mv.z, gv.z, r, wd, a);
        lars_elem(pv.w, mv.w, gv.w, r, wd, a);
        reinterpret_cast<float4*>(a.m)[q0 + i] = mv;
        store_all_ranks(sa, v0 + i, pv);
      }
      if (threadIdx.x < tail) {
        const size_t e = (size_t)start + (size_t)nv * 4 + threadIdx.x, eq = e - sa.lo;
        float pe = a.p[e], me = a.m[eq];
        lars_elem(pe, me, a.g[eq], r, wd, a);
        a.m[eq] = me;
        store_all_ranks1(sa, e, pe);
      }
    }
  }
  // every parameter slice has landed everywhere
  block_barrier_all_ranks(sa.sig, rank, world, ++epoch);
  if (a.zero_grad) {
    uint4* mine = reinterpret_cast<uint4*>(sa.grads.p[rank]);
    for (size_t j = (size_t)blockIdx.x * kLwThreads + threadIdx.x; j < sa.n_vec; j += (size_t)gridDim.x * kLwThreads)
      mine[j] = make_uint4(0u, 0u, 0u, 0u);
  }
  if (threadIdx.x == 0) barrier_epoch_store(sa.sig, rank, epoch);
}

template <bool kBf16, bool kLamb>
int sharded_layerwise_launch_t(const ShardedLwArgs& a, dim3 grid, cudaStream_t stream) {
  sharded_layerwise_norms_kernel<kBf16, kLamb><<<grid, kLwThreads, 0, stream>>>(a);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  sharded_layerwise_apply_kernel<kLamb><<<grid, kLwThreads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

}  // namespace b2

extern "C" {

// One sharded FlatLAMB (lamb != 0) or FlatLARS update of one bucket on `stream`: the norms kernel, then the apply kernel, each
// on shard_grid(n_vec, world, max_blocks) CTAs.  n_vec: 16-byte vectors of the gradient bucket (4 fp32 or, with bf16, 8 bf16
// gradients each), a multiple of world; rank r owns elements [r * per, (r + 1) * per), per = n_vec / world x 4 (x 8).  `lw`
// holds this rank's table (sharded_layerwise_table), partials, tickets, ratios, state shards (and LARS's gradient workspace
// shard in g), of per elements, and the scalars; its p, sums and n are set here.  Returns cudaError_t as int;
// cudaErrorInvalidValue, without a launch, for a world outside 1..8, a rank outside [0, world), an n_vec that is not a
// multiple of world, a null pointer, or clipping / loss scaling (the sharded update has neither).
int b2_sharded_layerwise_launch(int lamb, int bf16, const PeerPtrs* grads, const PeerPtrs* params, const PeerPtrs* sums,
                                const b2::SignalPads* sig, const b2::LwArgs* lw, size_t n_vec, float scale, int rank, int world,
                                int max_blocks, cudaStream_t stream) {
  if (world < 1 || world > B2_MAX_RANKS || rank < 0 || rank >= world || n_vec % (size_t)world != 0) return (int)cudaErrorInvalidValue;
  if (grads == nullptr || params == nullptr || sums == nullptr || sig == nullptr || lw == nullptr) return (int)cudaErrorInvalidValue;
  for (int r = 0; r < world; ++r)
    if (grads->p[r] == nullptr || params->p[r] == nullptr || sums->p[r] == nullptr || sig->pad[r] == nullptr)
      return (int)cudaErrorInvalidValue;
  if (lw->m == nullptr || (lamb ? lw->v == nullptr : lw->g == nullptr) || lw->table == nullptr || lw->tickets == nullptr ||
      lw->ratios == nullptr || lw->n_tensors < 1 || lw->n_chunks < 0 || (lw->n_chunks > 0 && lw->partials == nullptr) ||
      lw->max_norm != 0.f || lw->grad_scale != nullptr)
    return (int)cudaErrorInvalidValue;
  b2::ShardedLwArgs a;
  std::memset(&a, 0, sizeof(a));
  a.grads = *grads; a.params = *params; a.sums = *sums; a.sig = *sig;
  a.lw = *lw;
  a.n_vec = n_vec;
  a.lw.n = n_vec / (size_t)world * (bf16 ? 8 : 4);
  a.lo = (size_t)rank * a.lw.n;
  a.lw.p = reinterpret_cast<float*>(params->p[rank]);
  a.lw.sums = reinterpret_cast<double*>(sums->p[rank]);
  a.scale = scale; a.rank = rank; a.world = world;
  const dim3 grid = shard_grid(n_vec, world, max_blocks);
  using namespace b2;
  if (bf16) return lamb ? sharded_layerwise_launch_t<true, true>(a, grid, stream) : sharded_layerwise_launch_t<true, false>(a, grid, stream);
  return lamb ? sharded_layerwise_launch_t<false, true>(a, grid, stream) : sharded_layerwise_launch_t<false, false>(a, grid, stream);
}

}  // extern "C"
