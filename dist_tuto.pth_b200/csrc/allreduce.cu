// Fused peer-memory all-reduce kernels for sm_90a (NVLink / NVSwitch).
//
// Replaces the reference's hot path  `dist.all_reduce(param.grad.data, SUM); param.grad.data /= size`
// per parameter tensor (train_dist.py:94-100, tuto.md:310-314)  with ONE kernel per flat bucket that
//   * reads / writes the peers' buffers directly (symmetric memory mapped on every rank),
//   * sums in fp32 in fixed rank order (bit-identical result on every rank),
//   * fuses the 1/world_size scale and the bf16<->fp32 casts (wire dtype may differ from local dtype),
//   * synchronises with device-side release/acquire flag barriers (no NCCL, no host sync).
// Variants (picked per message size by parallel/symm.py from a measured table):
//   one-shot : every rank reads the whole buffer of every peer           (latency-optimal, <= ~256 KB)
//   two-shot : reduce-scatter (rank r owns slice r) + push all-gather    (2(N-1)/N * M bytes per GPU)
//   NVLS     : multimem.ld_reduce + multimem.st on a multicast address   (the switch does the sum)
//   LL       : flag-in-data push for small messages -- every rank STORES its vectors into every peer's inbox as 16-byte
//              lines {d0, epoch, d1, epoch} and reduces out of its own memory: no barrier, ONE NVLink crossing on the
//              critical path (the barrier variants need a flag crossing plus a load round trip)
//
// Work mapping invariant: element-vector j of a slice is always handled by the same (block, thread) on
// every rank and in every phase, which is what makes the *per-block* cross-GPU barriers sufficient.
//
// The same three data movements serve six collectives, selected by the OP template parameter:
//   SUM / PRODUCT / MAX / MIN : fp32 accumulator combined in rank order; `root` >= 0 makes it a reduce (only the root
//                               stores its output; every rank still runs every barrier and every LL push)
//   BCAST                     : raw 16-byte copies of the root's vectors (any dtype; never through the fp32 accumulator,
//                               so -0, subnormals, NaN payloads and integers survive)
//   GATHER                    : raw copies; rank r's input (n_vec / world vectors) lands at vector r * n_vec / world
// Every rank of one call runs the same barrier sequence whatever the op and root, so calls of any kind may follow each
// other on one buffer, signal pad and inbox.
#include <cstdio>
#include <cstring>
#include "common.cuh"

namespace b2 {

enum : int { kSum = 0, kProd = 1, kMax = 2, kMin = 3, kBcast = 4, kGather = 5 };

// The combine step of a reduction: identity, one fp32 combine, and the final scale (SUM only; the launcher refuses a
// scale for the other ops, and skipping the multiply keeps their results bit-exact under --use_fast_math).
template <int OP>
struct Op;
template <>
struct Op<kSum> {
  static constexpr float kIdentity = 0.f;
  __device__ static __forceinline__ float combine(float a, float b) { return a + b; }
  __device__ static __forceinline__ float fin(float a, float s) { return a * s; }
};
template <>
struct Op<kProd> {
  static constexpr float kIdentity = 1.f;
  __device__ static __forceinline__ float combine(float a, float b) { return a * b; }
  __device__ static __forceinline__ float fin(float a, float) { return a; }
};
// IEEE 754-2019 maximum / minimum: NaN if either term is NaN (max.NaN / min.NaN), and -0 < +0.
template <>
struct Op<kMax> {
  static constexpr float kIdentity = -__builtin_huge_valf();
  __device__ static __forceinline__ float combine(float a, float b) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
  }
  __device__ static __forceinline__ float fin(float a, float) { return a; }
};
template <>
struct Op<kMin> {
  static constexpr float kIdentity = __builtin_huge_valf();
  __device__ static __forceinline__ float combine(float a, float b) {
    float r;
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
  }
  __device__ static __forceinline__ float fin(float a, float) { return a; }
};

template <bool BF16>
struct Wire;  // one "vec" = 16 bytes on the wire

template <>
struct Wire<false> {                      // fp32 wire: 4 elements per vec
  static constexpr int kElems = 4;
  template <int OP>
  __device__ static __forceinline__ void zero(float* a) { a[0] = a[1] = a[2] = a[3] = Op<OP>::kIdentity; }
  template <int OP>
  __device__ static __forceinline__ void add(float* a, uint4 v) {
    a[0] = Op<OP>::combine(a[0], __uint_as_float(v.x)); a[1] = Op<OP>::combine(a[1], __uint_as_float(v.y));
    a[2] = Op<OP>::combine(a[2], __uint_as_float(v.z)); a[3] = Op<OP>::combine(a[3], __uint_as_float(v.w));
  }
  template <int OP>
  __device__ static __forceinline__ uint4 pack(const float* a, float s) {
    return make_uint4(__float_as_uint(Op<OP>::fin(a[0], s)), __float_as_uint(Op<OP>::fin(a[1], s)),
                      __float_as_uint(Op<OP>::fin(a[2], s)), __float_as_uint(Op<OP>::fin(a[3], s)));
  }
};
template <>
struct Wire<true> {                       // bf16 wire: 8 elements per vec, fp32 accumulation
  static constexpr int kElems = 8;
  template <int OP>
  __device__ static __forceinline__ void zero(float* a) {
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = Op<OP>::kIdentity;
  }
  template <int OP>
  __device__ static __forceinline__ void add(float* a, uint4 v) {
    const float t[8] = {bf16lo(v.x), bf16hi(v.x), bf16lo(v.y), bf16hi(v.y),
                        bf16lo(v.z), bf16hi(v.z), bf16lo(v.w), bf16hi(v.w)};
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = Op<OP>::combine(a[i], t[i]);
  }
  template <int OP>
  __device__ static __forceinline__ uint4 pack(const float* a, float s) {
    return make_uint4(pack_bf16x2(Op<OP>::fin(a[0], s), Op<OP>::fin(a[1], s)),
                      pack_bf16x2(Op<OP>::fin(a[2], s), Op<OP>::fin(a[3], s)),
                      pack_bf16x2(Op<OP>::fin(a[4], s), Op<OP>::fin(a[5], s)),
                      pack_bf16x2(Op<OP>::fin(a[6], s), Op<OP>::fin(a[7], s)));
  }
};

// local tensor <-> wire vec (local dtype is either the wire dtype or fp32)
template <bool BF16>
__device__ __forceinline__ uint4 load_local_as_wire(const void* base, size_t vec, bool local_f32) {
  if (!BF16 || !local_f32) return ld_cg_v4(reinterpret_cast<const uint4*>(base) + vec);
  const uint4 a = ld_cg_v4(reinterpret_cast<const uint4*>(base) + 2 * vec);
  const uint4 b = ld_cg_v4(reinterpret_cast<const uint4*>(base) + 2 * vec + 1);
  return make_uint4(pack_bf16x2(__uint_as_float(a.x), __uint_as_float(a.y)),
                    pack_bf16x2(__uint_as_float(a.z), __uint_as_float(a.w)),
                    pack_bf16x2(__uint_as_float(b.x), __uint_as_float(b.y)),
                    pack_bf16x2(__uint_as_float(b.z), __uint_as_float(b.w)));
}
template <bool BF16, int OP>
__device__ __forceinline__ void store_acc_local(void* base, size_t vec, const float* acc, float s, bool local_f32) {
  if (!BF16 || !local_f32 || OP != kSum) {
    st_cg_v4(reinterpret_cast<uint4*>(base) + vec, Wire<BF16>::template pack<OP>(acc, s));
  } else {  // bf16 wire, fp32 local (SUM only): keep the fp32 accumulator precision
    st_cg_v4(reinterpret_cast<uint4*>(base) + 2 * vec,
             make_uint4(__float_as_uint(acc[0] * s), __float_as_uint(acc[1] * s), __float_as_uint(acc[2] * s),
                        __float_as_uint(acc[3] * s)));
    st_cg_v4(reinterpret_cast<uint4*>(base) + 2 * vec + 1,
             make_uint4(__float_as_uint(acc[4] * s), __float_as_uint(acc[5] * s), __float_as_uint(acc[6] * s),
                        __float_as_uint(acc[7] * s)));
  }
}
template <bool BF16>
__device__ __forceinline__ void store_wire_local(void* base, size_t vec, uint4 w, bool local_f32) {
  if (!BF16 || !local_f32) {
    st_cg_v4(reinterpret_cast<uint4*>(base) + vec, w);
  } else {
    st_cg_v4(reinterpret_cast<uint4*>(base) + 2 * vec,
             make_uint4(__float_as_uint(bf16lo(w.x)), __float_as_uint(bf16hi(w.x)), __float_as_uint(bf16lo(w.y)),
                        __float_as_uint(bf16hi(w.y))));
    st_cg_v4(reinterpret_cast<uint4*>(base) + 2 * vec + 1,
             make_uint4(__float_as_uint(bf16lo(w.z)), __float_as_uint(bf16hi(w.z)), __float_as_uint(bf16lo(w.w)),
                        __float_as_uint(bf16hi(w.w))));
  }
}

struct ARArgs {
  PeerPtrs bufs;          // symmetric wire buffer of every rank
  SignalPads sig;         // signal pad of every rank (one pad per symmetric buffer)
  void* mc;               // multicast VA of the symmetric buffer (NVLS) or nullptr
  const void* src;        // optional local source (copied/cast into bufs.p[rank] first; GATHER: into slice rank)
  void* dst;              // optional local destination (else result stays in bufs.p[rank])
  size_t n_vec;           // 16-byte vectors on the wire (padded); GATHER: of the output, world x the per-rank input
  float scale;
  int rank, world;
  int src_f32, dst_f32;   // local dtypes: 1 = fp32, 0 = wire dtype
  PeerPtrs inbox;         // LL variant: every rank's inbox [2 parities][world sources][ll_cap vectors][2 lines of 16 B]
  size_t ll_cap;          // vectors per (parity, source) region of the inbox
  int root;               // reductions: -1 = every rank stores the result, else only this rank; BCAST: the source rank
};

constexpr int kThreads = 512;
constexpr int kUnroll = 2;        // peer-load variants: 2 x world 16-byte loads in flight per thread
constexpr int kUnrollNvls = 4;    // NVLS: one multimem.ld_reduce per vector

// Does this rank store its output?  Only a reduce (ROOT: a reduction with root >= 0) suppresses stores, never barriers.
// ROOT is a template parameter so that the all-reduce instances carry no root test at all.
template <bool ROOT>
__device__ __forceinline__ bool stores_output(const ARArgs& a) {
  return !ROOT || a.root == a.rank;
}

// ------------------------------------------------------------------------------------------ one-shot
// Reductions read vector v of every rank; BCAST reads it from the root only; GATHER reads it from its owner v / seg.
template <bool BF16, int OP, bool ROOT>
__global__ void __launch_bounds__(kThreads) allreduce_oneshot_kernel(ARArgs a) {
  using W = Wire<BF16>;
  constexpr bool kRaw = OP >= kBcast;
  const int rank = a.rank, world = a.world;
  uint32_t epoch = barrier_epoch_load(a.sig, rank);
  const size_t stride = (size_t)gridDim.x * kThreads;
  const size_t first = (size_t)blockIdx.x * kThreads + threadIdx.x;
  const size_t seg = a.n_vec / world;                   // GATHER: vectors per rank
  if (a.src != nullptr && (OP != kBcast || rank == a.root)) {
    uint4* stage = reinterpret_cast<uint4*>(a.bufs.p[rank]) + (OP == kGather ? (size_t)rank * seg : 0);
    for (size_t v = first; v < (OP == kGather ? seg : a.n_vec); v += stride)
      st_cg_v4(stage + v, load_local_as_wire<BF16>(a.src, v, a.src_f32));
  }
  block_barrier_all_ranks(a.sig, rank, world, ++epoch);          // every rank's data is in place
  const bool inplace = (a.dst == nullptr);
  void* out = inplace ? a.bufs.p[rank] : a.dst;
  const bool out_f32 = inplace ? false : (a.dst_f32 != 0);
  const bool store = stores_output<ROOT>(a);
  // block-uniform trip count (the in-place variant has a barrier inside the loop); identical on every rank
  for (size_t base0 = (size_t)blockIdx.x * kThreads; base0 < a.n_vec; base0 += stride * kUnroll) {
    const size_t base = base0 + threadIdx.x;
    float acc[kUnroll][W::kElems];
    uint4 raw[kUnroll][B2_MAX_RANKS];
    if constexpr (kRaw) {
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const size_t v = base + (size_t)u * stride;
        const int from = OP == kBcast ? a.root : (int)(v / seg);
        if (v < a.n_vec) raw[u][0] = ld_cg_v4(reinterpret_cast<const uint4*>(a.bufs.p[from]) + v);
      }
    } else {
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const size_t v = base + (size_t)u * stride;
#pragma unroll
        for (int r = 0; r < B2_MAX_RANKS; ++r)
          if (r < world && v < a.n_vec) raw[u][r] = ld_cg_v4(reinterpret_cast<const uint4*>(a.bufs.p[r]) + v);
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        W::template zero<OP>(acc[u]);
        const size_t v = base + (size_t)u * stride;
#pragma unroll
        for (int r = 0; r < B2_MAX_RANKS; ++r)
          if (r < world && v < a.n_vec) W::template add<OP>(acc[u], raw[u][r]);
      }
    }
    if (inplace) block_barrier_all_ranks(a.sig, rank, world, ++epoch);   // all peers finished reading this pass
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const size_t v = base + (size_t)u * stride;
      if (v < a.n_vec && store) {
        if constexpr (kRaw) st_cg_v4(reinterpret_cast<uint4*>(out) + v, raw[u][0]);
        else store_acc_local<BF16, OP>(out, v, acc[u], a.scale, out_f32);
      }
    }
  }
  if (!inplace) block_barrier_all_ranks(a.sig, rank, world, ++epoch);    // staging may be overwritten now
  if (threadIdx.x == 0) barrier_epoch_store(a.sig, rank, epoch);
}

// ------------------------------------------------------------------------------------------ two-shot / NVLS
// Slice s = vectors [s*slice, (s+1)*slice) is reduced by rank s and pushed to every rank (a reduce pushes it to the root
// only).  BCAST: rank s loads slice s from the root and pushes it; GATHER: rank s pushes its own input, staged at slice s.
template <bool BF16, bool NVLS, int OP, bool ROOT>
__global__ void __launch_bounds__(kThreads) allreduce_twoshot_kernel(ARArgs a) {
  using W = Wire<BF16>;
  constexpr bool kRaw = OP >= kBcast;
  const int rank = a.rank, world = a.world;
  uint32_t epoch = barrier_epoch_load(a.sig, rank);
  const size_t slice = a.n_vec / world;                 // host pads n_vec to a multiple of world
  const size_t stride = (size_t)gridDim.x * kThreads;
  const size_t first = (size_t)blockIdx.x * kThreads + threadIdx.x;
  if (a.src != nullptr && (OP != kBcast || rank == a.root)) {
    for (int s = 0; s < world; ++s) {
      if (OP == kGather && s != rank) continue;
      for (size_t j = first; j < slice; j += stride) {
        const size_t v = (size_t)s * slice + j;
        st_cg_v4(reinterpret_cast<uint4*>(a.bufs.p[rank]) + v,
                 load_local_as_wire<BF16>(a.src, OP == kGather ? j : v, a.src_f32));
      }
    }
  }
  block_barrier_all_ranks(a.sig, rank, world, ++epoch);
  const size_t off = (size_t)rank * slice;
  constexpr int U = NVLS ? kUnrollNvls : kUnroll;
  for (size_t base = first; base < slice; base += stride * U) {
    if constexpr (NVLS) {
      uint4 red[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t j = base + (size_t)u * stride;
        if (j < slice) {
          const uint4* p = reinterpret_cast<const uint4*>(a.mc) + off + j;
          if (BF16) {
            red[u] = multimem_ld_reduce_bf16x8(p);
          } else {
            float4 f = multimem_ld_reduce_f32x4(p);
            red[u] = make_uint4(__float_as_uint(f.x), __float_as_uint(f.y), __float_as_uint(f.z), __float_as_uint(f.w));
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t j = base + (size_t)u * stride;
        if (j < slice) {
          float acc[W::kElems];
          W::template zero<OP>(acc);
          W::template add<OP>(acc, red[u]);
          multimem_st_v4(reinterpret_cast<uint4*>(a.mc) + off + j, W::template pack<OP>(acc, a.scale));
        }
      }
    } else {
      uint4 raw[kUnroll][B2_MAX_RANKS];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const size_t j = base + (size_t)u * stride;
        if constexpr (kRaw) {
          if (j < slice) raw[u][0] = ld_cg_v4(reinterpret_cast<const uint4*>(a.bufs.p[OP == kBcast ? a.root : rank]) + off + j);
        } else {
#pragma unroll
          for (int r = 0; r < B2_MAX_RANKS; ++r)
            if (r < world && j < slice) raw[u][r] = ld_cg_v4(reinterpret_cast<const uint4*>(a.bufs.p[r]) + off + j);
        }
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const size_t j = base + (size_t)u * stride;
        if (j < slice) {
          uint4 o;
          if constexpr (kRaw) {
            o = raw[u][0];
          } else {
            float acc[W::kElems];
            W::template zero<OP>(acc);
#pragma unroll
            for (int r = 0; r < B2_MAX_RANKS; ++r)
              if (r < world) W::template add<OP>(acc, raw[u][r]);
            o = W::template pack<OP>(acc, a.scale);
          }
#pragma unroll
          for (int r = 0; r < B2_MAX_RANKS; ++r)
            if (r < world && (!ROOT || r == a.root)) st_cg_v4(reinterpret_cast<uint4*>(a.bufs.p[r]) + off + j, o);
        }
      }
    }
  }
  block_barrier_all_ranks(a.sig, rank, world, ++epoch);          // every slice has landed everywhere
  if (a.dst != nullptr && stores_output<ROOT>(a)) {
    for (int s = 0; s < world; ++s)
      for (size_t j = first; j < slice; j += stride) {
        const size_t v = (size_t)s * slice + j;
        store_wire_local<BF16>(a.dst, v, ld_cg_v4(reinterpret_cast<const uint4*>(a.bufs.p[rank]) + v), a.dst_f32);
      }
  }
  if (a.src != nullptr) block_barrier_all_ranks(a.sig, rank, world, ++epoch);  // staging reusable (eager path)
  if (threadIdx.x == 0) barrier_epoch_store(a.sig, rank, epoch);
}

// ------------------------------------------------------------------------------------------ LL (flag-in-data push)
// Every vector is handled by the same (block, thread) on all ranks and each block keeps its own call counter (the signal
// pad's per-block epoch word, shared with the barrier variants, which only ever compare epochs with >=), so sender and
// receiver of a line agree on epoch and parity without any cross-block coordination.  Parity double-buffers the inbox: a
// peer can write my parity-p region of block b again only two participations of block b later, which needs my lines of the
// participation in between, which I store after I finished reading parity p (same argument as sgd_device.cuh, model-checked
// in tests/test_protocol_models.py).  That needs the vector -> block map to be the same in every call on an inbox, so the
// launcher sizes the LL grid by the pushed vectors alone.  epoch 0 never occurs as a flag: counters are pre-incremented, the
// inbox starts zeroed, and the one epoch in 2^32 that wraps to 0 uses flag 1 (epoch 1 has the other parity).
// Every op pushes and waits for the same lines: BCAST keeps the root's line (the others are the acknowledgements the parity
// argument needs), GATHER stores source r's line at vector r * n_vec / world instead of combining it.
template <bool BF16, int OP, bool ROOT>
__global__ void __launch_bounds__(kThreads) allreduce_ll_kernel(ARArgs a) {
  using W = Wire<BF16>;
  const int rank = a.rank, world = a.world;
  const uint32_t epoch = barrier_epoch_load(a.sig, rank) + 1u;
  const uint32_t flag = epoch == 0u ? 1u : epoch;                     // 0 is "never written"
  const size_t par = (size_t)(epoch & 1u);
  const size_t stride = (size_t)gridDim.x * kThreads;
  const size_t n_push = OP == kGather ? a.n_vec / world : a.n_vec;    // vectors each rank pushes
  const void* in_local = a.src != nullptr ? a.src
                                          : reinterpret_cast<const uint4*>(a.bufs.p[rank]) + (OP == kGather ? rank * n_push : 0);
  const bool in_f32 = a.src != nullptr && a.src_f32 != 0;
  void* out = a.dst != nullptr ? a.dst : a.bufs.p[rank];
  const bool out_f32 = a.dst != nullptr && a.dst_f32 != 0;
  const bool store = stores_output<ROOT>(a);
  for (size_t v = (size_t)blockIdx.x * kThreads + threadIdx.x; v < n_push; v += stride) {
    const uint4 mine = load_local_as_wire<BF16>(in_local, v, in_f32);
    const uint4 l0 = make_uint4(mine.x, flag, mine.y, flag), l1 = make_uint4(mine.z, flag, mine.w, flag);
    const size_t line = ((par * (size_t)world + (size_t)rank) * a.ll_cap + v) * 2;
#pragma unroll
    for (int i = 1; i < B2_MAX_RANKS; ++i) {
      if (i < world) {
        int r = rank + i;
        if (r >= world) r -= world;
        uint4* d = reinterpret_cast<uint4*>(a.inbox.p[r]) + line;
        st_volatile_v4(d, l0);
        st_volatile_v4(d + 1, l1);
      }
    }
    float acc[W::kElems];
    if constexpr (OP < kBcast) W::template zero<OP>(acc);
    uint4 kept = mine;                                                // BCAST: the root's vector
    const uint4* in = reinterpret_cast<const uint4*>(a.inbox.p[rank]);
#pragma unroll
    for (int r = 0; r < B2_MAX_RANKS; ++r) {
      if (r < world) {
        uint4 w;
        if (r == rank) {
          w = mine;
        } else {
          const uint4* src = in + ((par * (size_t)world + (size_t)r) * a.ll_cap + v) * 2;
          uint4 q0, q1;
          unsigned long long spins = 0;
          for (;;) {
            q0 = ld_volatile_v4(src);
            q1 = ld_volatile_v4(src + 1);
            if (q0.y == flag && q0.w == flag && q1.y == flag && q1.w == flag) break;
            if (++spins > B2_SPIN_LIMIT) {
              printf("[b200dist] LL all-reduce: rank %d timed out waiting for rank %d (block %d, epoch %u)\n", rank, r, (int)blockIdx.x, flag);
              __trap();
            }
          }
          w = make_uint4(q0.x, q0.z, q1.x, q1.z);
        }
        if constexpr (OP == kGather) st_cg_v4(reinterpret_cast<uint4*>(out) + (size_t)r * n_push + v, w);
        else if constexpr (OP == kBcast) kept = r == a.root ? w : kept;
        else W::template add<OP>(acc, w);                             // fixed rank order => bit-identical on every rank
      }
    }
    if constexpr (OP == kBcast) st_cg_v4(reinterpret_cast<uint4*>(out) + v, kept);
    else if constexpr (OP != kGather) {
      if (store) store_acc_local<BF16, OP>(out, v, acc, a.scale, out_f32);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) barrier_epoch_store(a.sig, rank, epoch);
}

// ------------------------------------------------------------------------------------------ barrier only
__global__ void __launch_bounds__(32) barrier_kernel(SignalPads sig, int rank, int world) {
  uint32_t epoch = barrier_epoch_load(sig, rank);
  block_barrier_all_ranks(sig, rank, world, ++epoch);
  if (threadIdx.x == 0) barrier_epoch_store(sig, rank, epoch);
}

}  // namespace b2

namespace b2 {

template <bool BF16, int OP, bool ROOT>
void launch_kernel(int variant, dim3 grid, const ARArgs& a, cudaStream_t stream) {
  if (variant == 0) allreduce_oneshot_kernel<BF16, OP, ROOT><<<grid, kThreads, 0, stream>>>(a);
  else if (variant == 1) allreduce_twoshot_kernel<BF16, false, OP, ROOT><<<grid, kThreads, 0, stream>>>(a);
  else if (variant == 3) allreduce_ll_kernel<BF16, OP, ROOT><<<grid, kThreads, 0, stream>>>(a);
  else if constexpr (OP == kSum && !ROOT) allreduce_twoshot_kernel<BF16, true, kSum, false><<<grid, kThreads, 0, stream>>>(a);
}

template <int OP>
void launch_op(int variant, int bf16, dim3 grid, const ARArgs& a, cudaStream_t stream) {
  if constexpr (OP < kBcast) {
    if (a.root >= 0) return bf16 ? launch_kernel<true, OP, true>(variant, grid, a, stream)
                                 : launch_kernel<false, OP, true>(variant, grid, a, stream);
    if (bf16) return launch_kernel<true, OP, false>(variant, grid, a, stream);
  }
  launch_kernel<false, OP, false>(variant, grid, a, stream);
}

}  // namespace b2

// ============================================================================================ launchers
extern "C" {

// variant: 0 one-shot, 1 two-shot, 2 NVLS, 3 LL (needs inbox / ll_cap).  op: 0 SUM, 1 PRODUCT, 2 MAX, 3 MIN, 4 broadcast
// from `root`, 5 all-gather; a reduction with root >= 0 is a reduce to that rank.  Returns cudaError_t as int;
// cudaErrorInvalidValue, without a launch, for an unknown variant or op, a world outside 1..8, a rank outside [0, world), a
// root outside [-1, world) (a broadcast needs one, an all-gather takes none), a scale other than 1, fp32 locals over a bf16
// wire or NVLS for any op but SUM, a bf16 wire for the raw moves, a two-shot / NVLS / all-gather n_vec that is not a
// multiple of world (the remainder would be left out) or an LL message larger than the inbox.
int b2_allreduce_launch(int variant, int bf16, const PeerPtrs* bufs, const b2::SignalPads* sig, void* mc,
                        const void* src, int src_f32, void* dst, int dst_f32, size_t n_vec, float scale,
                        int rank, int world, int max_blocks, const PeerPtrs* inbox, size_t ll_cap, int op, int root,
                        cudaStream_t stream) {
  if (variant < 0 || variant > 3 || world < 1 || world > B2_MAX_RANKS || rank < 0 || rank >= world)
    return (int)cudaErrorInvalidValue;
  if (op < b2::kSum || op > b2::kGather || root < -1 || root >= world) return (int)cudaErrorInvalidValue;
  if (op == b2::kBcast ? root < 0 : (op == b2::kGather && root >= 0)) return (int)cudaErrorInvalidValue;
  if (op != b2::kSum && (scale != 1.f || src_f32 || dst_f32)) return (int)cudaErrorInvalidValue;
  if (variant == 2 && (op != b2::kSum || root >= 0)) return (int)cudaErrorInvalidValue;   // NVLS: the SUM all-reduce only
  if (op >= b2::kBcast && bf16) return (int)cudaErrorInvalidValue;
  if ((variant == 1 || variant == 2 || op == b2::kGather) && n_vec % (size_t)world != 0)
    return (int)cudaErrorInvalidValue;                                     // slice = n_vec / world
  const size_t n_push = op == b2::kGather ? n_vec / world : n_vec;        // LL: vectors each rank pushes
  b2::ARArgs a;
  memset(&a.inbox, 0, sizeof(a.inbox));
  a.ll_cap = 0;
  a.bufs = *bufs; a.sig = *sig; a.mc = mc; a.src = src; a.dst = dst; a.n_vec = n_vec; a.scale = scale;
  a.rank = rank; a.world = world; a.src_f32 = src_f32; a.dst_f32 = dst_f32; a.root = root;
  if (variant == 3) {
    if (inbox == nullptr || ll_cap < n_push) return (int)cudaErrorInvalidValue;
    a.inbox = *inbox;
    a.ll_cap = ll_cap;
  }
  if (variant == 2 && mc == nullptr) return (int)cudaErrorInvalidValue;
  if (max_blocks <= 0 || max_blocks > B2_MAX_BLOCKS) max_blocks = B2_MAX_BLOCKS;
  const size_t work = variant == 0 ? n_vec : variant == 3 ? n_push : n_vec / world;
  size_t blocks = (work + b2::kThreads - 1) / b2::kThreads;
  if (variant == 1 || variant == 2) blocks = (blocks + 1) / 2;
  if (blocks < 1) blocks = 1;
  // LL: the grid follows the message, never the per-call cap.  Vector v belongs to block (v / kThreads) % grid, whose own epoch
  // word gives the line's flag and parity; if the cap could change the grid between two calls on one inbox, v could move to a
  // block whose next flag equals the one its line already holds, and that stale line would be accepted.  n_push <= ll_cap keeps
  // the grid at ceil(4096 / 512) = 8 CTAs for the inbox parallel/symm.py allocates, so v's block is v / kThreads in every op.
  const size_t cap = variant == 3 ? (size_t)B2_MAX_BLOCKS : (size_t)max_blocks;
  if (blocks > cap) blocks = cap;
  const dim3 grid((unsigned)blocks);
  switch (op) {
    case b2::kSum: b2::launch_op<b2::kSum>(variant, bf16, grid, a, stream); break;
    case b2::kProd: b2::launch_op<b2::kProd>(variant, bf16, grid, a, stream); break;
    case b2::kMax: b2::launch_op<b2::kMax>(variant, bf16, grid, a, stream); break;
    case b2::kMin: b2::launch_op<b2::kMin>(variant, bf16, grid, a, stream); break;
    case b2::kBcast: b2::launch_op<b2::kBcast>(variant, bf16, grid, a, stream); break;
    default: b2::launch_op<b2::kGather>(variant, bf16, grid, a, stream); break;
  }
  return (int)cudaGetLastError();
}

int b2_barrier_launch(const b2::SignalPads* sig, int rank, int world, cudaStream_t stream) {
  b2::barrier_kernel<<<1, 32, 0, stream>>>(*sig, rank, world);
  return (int)cudaGetLastError();
}

}  // extern "C"
