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
//   GATHER                    : raw copies; rank r's input (n_vec / world vectors) lands at vector r * n_vec / world of every
//                               rank's output (all-gather) or, with `root` >= 0, of the root's only (gather)
//   SCATTER                   : raw copies; the root's input holds world segments of n_vec / world vectors and rank r
//                               receives segment r (at vector r * n_vec / world of its symmetric buffer when in place)
// Every rank of one call runs the same barrier sequence whatever the op and root, so calls of any kind may follow each
// other on one buffer, signal pad and inbox.
// Reduce-scatter and all-to-all have kernels of their own (segments_pull_kernel, segments_ll_kernel: a pull with barriers
// and an LL push) on the same lanes, per-block epoch words and inbox, so they too may follow any call on one buffer.
// The all-to-all with variable segments (alltoallv_kernel: rounds of a fixed chunk through a double-buffered staging window)
// uses the same signal pads and per-block epoch words and ends with the same final barrier, so it too may follow any call.
#include <cstdio>
#include <cstring>
#include <cuda_fp16.h>
#include <type_traits>
#include "common.cuh"

namespace b2 {

enum : int { kSum = 0, kProd = 1, kMax = 2, kMin = 3, kBcast = 4, kGather = 5, kScatter = 6 };

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

// Lane types: how one 16-byte vector on the wire splits into accumulator lanes, per dtype class.  Every lane type has
// `Acc` (the lane's accumulator type), kElems lanes per vector, zero<OP> (the identity), add<OP> (combine one vector into the
// lanes) and pack<OP> (the lanes back to a vector).  kF32Local: the local tensor may be fp32 over this wire (bf16 SUM only);
// kNvls: the switch can reduce this wire (multimem.ld_reduce).  Only fp32 / bf16 take a scale; the launcher refuses one for
// the others, whose pack ignores it.
enum : int { kF32 = 0, kBF16 = 1, kF16 = 2, kF64 = 3, kI8 = 4, kU8 = 5, kI32 = 6, kI64 = 7, kBool = 8 };

struct LaneF32 {                          // fp32 wire: 4 elements per vec
  using Acc = float;
  static constexpr int kElems = 4;
  static constexpr bool kF32Local = false, kNvls = true;
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
struct LaneBF16 {                         // bf16 wire: 8 elements per vec, fp32 accumulation
  using Acc = float;
  static constexpr int kElems = 8;
  static constexpr bool kF32Local = true, kNvls = true;
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

__device__ __forceinline__ float f16lo(uint32_t w) { return __half2float(__ushort_as_half((unsigned short)(w & 0xffffu))); }
__device__ __forceinline__ float f16hi(uint32_t w) { return __half2float(__ushort_as_half((unsigned short)(w >> 16))); }
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

struct LaneF16 {                          // fp16 wire: 8 elements per vec, fp32 accumulation, one RN-even rounding at the end
  using Acc = float;
  static constexpr int kElems = 8;
  static constexpr bool kF32Local = false, kNvls = false;
  template <int OP>
  __device__ static __forceinline__ void zero(float* a) {
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = Op<OP>::kIdentity;
  }
  template <int OP>
  __device__ static __forceinline__ void add(float* a, uint4 v) {
    const float t[8] = {f16lo(v.x), f16hi(v.x), f16lo(v.y), f16hi(v.y), f16lo(v.z), f16hi(v.z), f16lo(v.w), f16hi(v.w)};
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = Op<OP>::combine(a[i], t[i]);
  }
  template <int OP>
  __device__ static __forceinline__ uint4 pack(const float* a, float) {
    return make_uint4(pack_f16x2(a[0], a[1]), pack_f16x2(a[2], a[3]), pack_f16x2(a[4], a[5]), pack_f16x2(a[6], a[7]));
  }
};

// fp64: 2 lanes, combined in fp64.  MAX / MIN are IEEE 754-2019 maximum / minimum by hand (PTX has no max.NaN.f64): NaN if
// either term is NaN, returned as 0x7FFFFFFFFFFFFFFF like the fp32 kernels' 0x7FFFFFFF, and -0 < +0.
struct LaneF64 {
  using Acc = double;
  static constexpr int kElems = 2;
  static constexpr bool kF32Local = false, kNvls = false;
  template <int OP>
  __device__ static __forceinline__ double combine(double a, double b) {
    if constexpr (OP == kSum) return a + b;
    else if constexpr (OP == kProd) return a * b;
    else {
      const unsigned long long ia = __double_as_longlong(a), ib = __double_as_longlong(b);
      const unsigned long long kAbs = 0x7FFFFFFFFFFFFFFFull, kInf = 0x7FF0000000000000ull;
      if ((ia & kAbs) > kInf || (ib & kAbs) > kInf) return __longlong_as_double((long long)kAbs);
      if (a == b) return __longlong_as_double((long long)(OP == kMax ? ia & ib : ia | ib));   // +-0: the sign decides
      return (OP == kMax ? a > b : a < b) ? a : b;
    }
  }
  template <int OP>
  __device__ static __forceinline__ void zero(double* a) {
    a[0] = a[1] = OP == kSum ? 0.0 : OP == kProd ? 1.0 : OP == kMax ? -__builtin_huge_val() : __builtin_huge_val();
  }
  template <int OP>
  __device__ static __forceinline__ void add(double* a, uint4 v) {
    double t[2];
    memcpy(t, &v, 16);
    a[0] = combine<OP>(a[0], t[0]);
    a[1] = combine<OP>(a[1], t[1]);
  }
  template <int OP>
  __device__ static __forceinline__ uint4 pack(const double* a, float) {
    uint4 v;
    memcpy(&v, a, 16);
    return v;
  }
};

// int32 / int64: two's-complement lanes (4 or 2 per vec).  SUM and PRODUCT wrap mod 2^bits (unsigned arithmetic, as NCCL
// does), MAX / MIN compare signed.
template <class U, class S>
struct LaneInt {
  using Acc = U;
  static constexpr int kElems = 16 / sizeof(U);
  static constexpr bool kF32Local = false, kNvls = false;
  template <int OP>
  __device__ static __forceinline__ U combine(U a, U b) {
    if constexpr (OP == kSum) return a + b;
    else if constexpr (OP == kProd) return a * b;
    else if constexpr (OP == kMax) return (S)a > (S)b ? a : b;
    else return (S)a < (S)b ? a : b;
  }
  template <int OP>
  __device__ static __forceinline__ void zero(U* a) {
    const U top = (U)1 << (8 * sizeof(U) - 1);                            // the most negative value
#pragma unroll
    for (int i = 0; i < kElems; ++i) a[i] = OP == kSum ? (U)0 : OP == kProd ? (U)1 : OP == kMax ? top : top - 1;
  }
  template <int OP>
  __device__ static __forceinline__ void add(U* a, uint4 v) {
    U t[kElems];
    memcpy(t, &v, 16);
#pragma unroll
    for (int i = 0; i < kElems; ++i) a[i] = combine<OP>(a[i], t[i]);
  }
  template <int OP>
  __device__ static __forceinline__ uint4 pack(const U* a, float) {
    uint4 v;
    memcpy(&v, a, 16);
    return v;
  }
};
using LaneI32 = LaneInt<uint32_t, int32_t>;
using LaneI64 = LaneInt<unsigned long long, long long>;

// int8 / uint8 (and bool): 16 bytes as four packed 32-bit words of byte SIMD.  SUM (__vadd4) and PRODUCT (per byte) wrap
// mod 256 and are the same bits for both signs, so uint8 takes the int8 instances for them; MAX / MIN compare signed or
// unsigned bytes.
template <bool SIGNED>
struct LaneI8 {
  using Acc = uint32_t;
  static constexpr int kElems = 4;
  static constexpr bool kF32Local = false, kNvls = false;
  template <int OP>
  __device__ static __forceinline__ uint32_t combine(uint32_t a, uint32_t b) {
    if constexpr (OP == kSum) {
      return __vadd4(a, b);
    } else if constexpr (OP == kProd) {
      uint32_t p[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) p[i] = __byte_perm(a, 0u, 0x4440u + i) * __byte_perm(b, 0u, 0x4440u + i);
      return __byte_perm(__byte_perm(p[0], p[1], 0x0040u), __byte_perm(p[2], p[3], 0x0040u), 0x5410u);
    } else {
      uint32_t m[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {                                  // byte i, sign- or zero-extended to 32 bits
        const uint32_t sel = SIGNED ? (0x8880u | (i << 12) | (i << 8) | (i << 4)) + i : 0x4440u + i;
        const uint32_t x = __byte_perm(a, 0u, sel), y = __byte_perm(b, 0u, sel);
        m[i] = OP == kMax ? (SIGNED ? (uint32_t)max((int)x, (int)y) : max(x, y)) : (SIGNED ? (uint32_t)min((int)x, (int)y) : min(x, y));
      }
      return __byte_perm(__byte_perm(m[0], m[1], 0x0040u), __byte_perm(m[2], m[3], 0x0040u), 0x5410u);
    }
  }
  template <int OP>
  __device__ static __forceinline__ void zero(uint32_t* a) {
    a[0] = a[1] = a[2] = a[3] = OP == kSum ? 0u : OP == kProd ? 0x01010101u
                              : OP == kMax ? (SIGNED ? 0x80808080u : 0u) : (SIGNED ? 0x7F7F7F7Fu : 0xFFFFFFFFu);
  }
  template <int OP>
  __device__ static __forceinline__ void add(uint32_t* a, uint4 v) {
    a[0] = combine<OP>(a[0], v.x); a[1] = combine<OP>(a[1], v.y); a[2] = combine<OP>(a[2], v.z); a[3] = combine<OP>(a[3], v.w);
  }
  template <int OP>
  __device__ static __forceinline__ uint4 pack(const uint32_t* a, float) { return make_uint4(a[0], a[1], a[2], a[3]); }
};

// local tensor <-> wire vec (local dtype is either the wire dtype or, on a kF32Local wire, fp32)
template <class L>
__device__ __forceinline__ uint4 load_local_as_wire(const void* base, size_t vec, bool local_f32) {
  if (!L::kF32Local || !local_f32) return ld_cg_v4(reinterpret_cast<const uint4*>(base) + vec);
  const uint4 a = ld_cg_v4(reinterpret_cast<const uint4*>(base) + 2 * vec);
  const uint4 b = ld_cg_v4(reinterpret_cast<const uint4*>(base) + 2 * vec + 1);
  return make_uint4(pack_bf16x2(__uint_as_float(a.x), __uint_as_float(a.y)),
                    pack_bf16x2(__uint_as_float(a.z), __uint_as_float(a.w)),
                    pack_bf16x2(__uint_as_float(b.x), __uint_as_float(b.y)),
                    pack_bf16x2(__uint_as_float(b.z), __uint_as_float(b.w)));
}
template <class L, int OP>
__device__ __forceinline__ void store_acc_local(void* base, size_t vec, const typename L::Acc* acc, float s, bool local_f32) {
  if constexpr (!L::kF32Local) {
    st_cg_v4(reinterpret_cast<uint4*>(base) + vec, L::template pack<OP>(acc, s));
  } else if (!local_f32 || OP != kSum) {
    st_cg_v4(reinterpret_cast<uint4*>(base) + vec, L::template pack<OP>(acc, s));
  } else {  // bf16 wire, fp32 local (SUM only): keep the fp32 accumulator precision
    st_cg_v4(reinterpret_cast<uint4*>(base) + 2 * vec,
             make_uint4(__float_as_uint(acc[0] * s), __float_as_uint(acc[1] * s), __float_as_uint(acc[2] * s),
                        __float_as_uint(acc[3] * s)));
    st_cg_v4(reinterpret_cast<uint4*>(base) + 2 * vec + 1,
             make_uint4(__float_as_uint(acc[4] * s), __float_as_uint(acc[5] * s), __float_as_uint(acc[6] * s),
                        __float_as_uint(acc[7] * s)));
  }
}
template <class L>
__device__ __forceinline__ void store_wire_local(void* base, size_t vec, uint4 w, bool local_f32) {
  if (!L::kF32Local || !local_f32) {
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
  void* dst;              // optional local destination (else result stays in bufs.p[rank]; SCATTER: in its slice rank)
  size_t n_vec;           // 16-byte vectors on the wire (padded); GATHER: of the output, SCATTER: of the root's input,
                          // world x the per-rank segment in both
  float scale;
  int rank, world;
  int src_f32, dst_f32;   // local dtypes: 1 = fp32, 0 = wire dtype
  PeerPtrs inbox;         // LL variant: every rank's inbox [2 parities][world sources][ll_cap vectors][2 lines of 16 B]
  size_t ll_cap;          // vectors per (parity, source) region of the inbox
  int root;               // reductions and GATHER: -1 = every rank stores the result, else only this rank; BCAST and
                          // SCATTER: the source rank
};

constexpr int kThreads = 512;
constexpr int kUnroll = 2;        // peer-load variants: 2 x world 16-byte loads in flight per thread
constexpr int kUnrollNvls = 4;    // NVLS: one multimem.ld_reduce per vector

// Does this rank store its output?  Only a reduce or a gather (ROOT: root >= 0) suppresses stores, never barriers.
// ROOT is a template parameter so that the all-reduce instances carry no root test at all.
template <bool ROOT>
__device__ __forceinline__ bool stores_output(const ARArgs& a) {
  return !ROOT || a.root == a.rank;
}

// Broadcast and scatter read the root's input only: the other ranks' src is never read (it is passed all the same, so that
// every rank runs the same barriers).
template <int OP>
constexpr bool kFromRoot = OP == kBcast || OP == kScatter;

// ------------------------------------------------------------------------------------------ one-shot
// Reductions read vector v of every rank; BCAST reads it from the root only; GATHER reads it from its owner v / seg (a gather:
// on the root only); SCATTER: rank r reads the seg vectors of slot r from the root.
template <class L, int OP, bool ROOT>
__global__ void __launch_bounds__(kThreads) allreduce_oneshot_kernel(ARArgs a) {
  using W = L;
  constexpr bool kRaw = OP >= kBcast;
  const int rank = a.rank, world = a.world;
  uint32_t epoch = barrier_epoch_load(a.sig, rank);
  const size_t stride = (size_t)gridDim.x * kThreads;
  const size_t first = (size_t)blockIdx.x * kThreads + threadIdx.x;
  const size_t seg = a.n_vec / world;                   // GATHER / SCATTER: vectors per rank
  const size_t n_out = OP == kScatter ? seg : a.n_vec;  // vectors this rank reads and stores
  if (a.src != nullptr && (!kFromRoot<OP> || rank == a.root)) {
    uint4* stage = reinterpret_cast<uint4*>(a.bufs.p[rank]) + (OP == kGather ? (size_t)rank * seg : 0);
    for (size_t v = first; v < (OP == kGather ? seg : a.n_vec); v += stride)
      st_cg_v4(stage + v, load_local_as_wire<L>(a.src, v, a.src_f32));
  }
  block_barrier_all_ranks(a.sig, rank, world, ++epoch);          // every rank's data is in place
  const bool inplace = (a.dst == nullptr);
  void* out = inplace ? reinterpret_cast<uint4*>(a.bufs.p[rank]) + (OP == kScatter ? (size_t)rank * seg : 0) : a.dst;
  const bool out_f32 = inplace ? false : (a.dst_f32 != 0);
  const bool store = stores_output<ROOT>(a);
  // block-uniform trip count (the in-place variant has a barrier inside the loop); identical on every rank
  for (size_t base0 = (size_t)blockIdx.x * kThreads; base0 < n_out; base0 += stride * kUnroll) {
    const size_t base = base0 + threadIdx.x;
    typename W::Acc acc[kUnroll][W::kElems];
    uint4 raw[kUnroll][B2_MAX_RANKS];
    if constexpr (kRaw) {
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const size_t v = base + (size_t)u * stride;
        const int from = OP == kGather ? (int)(v / seg) : a.root;
        const size_t at = OP == kScatter ? (size_t)rank * seg + v : v;
        if (v < n_out && store) raw[u][0] = ld_cg_v4(reinterpret_cast<const uint4*>(a.bufs.p[from]) + at);
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
      if (v < n_out && store) {
        if constexpr (kRaw) st_cg_v4(reinterpret_cast<uint4*>(out) + v, raw[u][0]);
        else store_acc_local<L, OP>(out, v, acc[u], a.scale, out_f32);
      }
    }
  }
  if (!inplace) block_barrier_all_ranks(a.sig, rank, world, ++epoch);    // staging may be overwritten now
  if (threadIdx.x == 0) barrier_epoch_store(a.sig, rank, epoch);
}

// ------------------------------------------------------------------------------------------ two-shot / NVLS
// Slice s = vectors [s*slice, (s+1)*slice) is reduced by rank s and pushed to every rank (a reduce pushes it to the root
// only).  BCAST: rank s loads slice s from the root and pushes it; GATHER: rank s pushes its own input, staged at slice s (a
// gather: to the root only); SCATTER: the root pushes slice s of its input into rank s's slice s, and rank s copies it out.
template <class L, bool NVLS, int OP, bool ROOT>
__global__ void __launch_bounds__(kThreads) allreduce_twoshot_kernel(ARArgs a) {
  using W = L;
  constexpr bool kRaw = OP >= kBcast;
  const int rank = a.rank, world = a.world;
  uint32_t epoch = barrier_epoch_load(a.sig, rank);
  const size_t slice = a.n_vec / world;                 // host pads n_vec to a multiple of world
  const size_t stride = (size_t)gridDim.x * kThreads;
  const size_t first = (size_t)blockIdx.x * kThreads + threadIdx.x;
  if (a.src != nullptr && (!kFromRoot<OP> || rank == a.root)) {
    for (int s = 0; s < world; ++s) {
      if (OP == kGather && s != rank) continue;
      for (size_t j = first; j < slice; j += stride) {
        const size_t v = (size_t)s * slice + j;
        st_cg_v4(reinterpret_cast<uint4*>(a.bufs.p[rank]) + v,
                 load_local_as_wire<L>(a.src, OP == kGather ? j : v, a.src_f32));
      }
    }
  }
  block_barrier_all_ranks(a.sig, rank, world, ++epoch);
  const size_t off = (size_t)rank * slice;
  constexpr int U = NVLS ? kUnrollNvls : kUnroll;
  for (size_t base = first; base < slice; base += stride * U) {
    if constexpr (OP == kScatter) {
      if (rank != a.root) break;                                  // only the root pushes; no barrier inside this loop
      uint4 raw[kUnroll][B2_MAX_RANKS];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const size_t j = base + (size_t)u * stride;
#pragma unroll
        for (int r = 0; r < B2_MAX_RANKS; ++r)
          if (r < world && r != rank && j < slice)
            raw[u][r] = ld_cg_v4(reinterpret_cast<const uint4*>(a.bufs.p[rank]) + (size_t)r * slice + j);
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const size_t j = base + (size_t)u * stride;
#pragma unroll
        for (int r = 0; r < B2_MAX_RANKS; ++r)
          if (r < world && r != rank && j < slice)
            st_cg_v4(reinterpret_cast<uint4*>(a.bufs.p[r]) + (size_t)r * slice + j, raw[u][r]);
      }
    } else if constexpr (NVLS) {
      uint4 red[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const size_t j = base + (size_t)u * stride;
        if (j < slice) {
          const uint4* p = reinterpret_cast<const uint4*>(a.mc) + off + j;
          if (std::is_same<L, LaneBF16>::value) {   // only the fp32 and bf16 lanes reach NVLS
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
          typename W::Acc acc[W::kElems];
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
            typename W::Acc acc[W::kElems];
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
    for (int s = 0; s < world; ++s) {
      if (OP == kScatter && s != rank) continue;
      for (size_t j = first; j < slice; j += stride) {
        const size_t v = (size_t)s * slice + j;
        store_wire_local<L>(a.dst, OP == kScatter ? j : v, ld_cg_v4(reinterpret_cast<const uint4*>(a.bufs.p[rank]) + v),
                               a.dst_f32);
      }
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
// argument needs), GATHER stores source r's line at vector r * n_vec / world instead of combining it (a gather: on the root
// only), and SCATTER is BCAST except that the root's line to rank r carries segment r of its input.
template <class L, int OP, bool ROOT>
__global__ void __launch_bounds__(kThreads) allreduce_ll_kernel(ARArgs a) {
  using W = L;
  const int rank = a.rank, world = a.world;
  const uint32_t epoch = barrier_epoch_load(a.sig, rank) + 1u;
  const uint32_t flag = epoch == 0u ? 1u : epoch;                     // 0 is "never written"
  const size_t par = (size_t)(epoch & 1u);
  const size_t stride = (size_t)gridDim.x * kThreads;
  const size_t n_push = OP == kGather || OP == kScatter ? a.n_vec / world : a.n_vec;    // vectors each rank pushes
  const void* in_local = a.src != nullptr ? a.src
                                          : reinterpret_cast<const uint4*>(a.bufs.p[rank]) + (OP == kGather ? rank * n_push : 0);
  const bool in_f32 = a.src != nullptr && a.src_f32 != 0;
  void* out = a.dst != nullptr ? a.dst : reinterpret_cast<uint4*>(a.bufs.p[rank]) + (OP == kScatter ? rank * n_push : 0);
  const bool out_f32 = a.dst != nullptr && a.dst_f32 != 0;
  const bool store = stores_output<ROOT>(a);
  for (size_t v = (size_t)blockIdx.x * kThreads + threadIdx.x; v < n_push; v += stride) {
    // SCATTER: the root's own segment; a non-root reads no input (its src may be any size) and pushes zeros
    const uint4 mine = OP == kScatter && rank != a.root
                           ? make_uint4(0u, 0u, 0u, 0u)
                           : load_local_as_wire<L>(in_local, OP == kScatter ? (size_t)rank * n_push + v : v, in_f32);
    const uint4 l0 = make_uint4(mine.x, flag, mine.y, flag), l1 = make_uint4(mine.z, flag, mine.w, flag);
    const size_t line = ((par * (size_t)world + (size_t)rank) * a.ll_cap + v) * 2;
#pragma unroll
    for (int i = 1; i < B2_MAX_RANKS; ++i) {
      if (i < world) {
        int r = rank + i;
        if (r >= world) r -= world;
        uint4* d = reinterpret_cast<uint4*>(a.inbox.p[r]) + line;
        if constexpr (OP == kScatter) {                               // the root's line to rank r carries segment r
          const uint4 w = rank == a.root ? load_local_as_wire<L>(in_local, (size_t)r * n_push + v, in_f32) : mine;
          st_volatile_v4(d, make_uint4(w.x, flag, w.y, flag));
          st_volatile_v4(d + 1, make_uint4(w.z, flag, w.w, flag));
        } else {
          st_volatile_v4(d, l0);
          st_volatile_v4(d + 1, l1);
        }
      }
    }
    typename W::Acc acc[W::kElems];
    if constexpr (OP < kBcast) W::template zero<OP>(acc);
    uint4 kept = mine;                                                // BCAST / SCATTER: the root's vector
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
        if constexpr (OP == kGather) {
          if (store) st_cg_v4(reinterpret_cast<uint4*>(out) + (size_t)r * n_push + v, w);
        } else if constexpr (kFromRoot<OP>) {
          kept = r == a.root ? w : kept;
        } else {
          W::template add<OP>(acc, w);                                // fixed rank order => bit-identical on every rank
        }
      }
    }
    if constexpr (kFromRoot<OP>) st_cg_v4(reinterpret_cast<uint4*>(out) + v, kept);
    else if constexpr (OP != kGather) {
      if (store) store_acc_local<L, OP>(out, v, acc, a.scale, out_f32);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) barrier_epoch_store(a.sig, rank, epoch);
}

// ------------------------------------------------------------------------------------------ reduce-scatter / all-to-all
// n_vec = world segments of seg = n_vec / world vectors on every rank.  Reduce-scatter (A2A false): rank r's output is
// segment r of the reduction, combined exactly as the all-reduce combines it (identity, then every rank's term in rank order,
// pack with scale 1), so it is bit for bit slice r of the all-reduce of the same inputs.  All-to-all (A2A true, raw 16-byte
// copies): segment p of rank r's output is segment r of rank p's input.  Vector j of every segment is handled by the same
// (block, thread) in every phase and on every rank, so the per-block barriers suffice.
//
// Pull: stage src into this rank's buffer (unless it is already there), barrier, load segment `rank` of every rank's buffer,
// store to dst (reduce-scatter in place: to segment `rank` of this rank's buffer, which no peer reads), barrier (the peers
// have finished reading this buffer, so the caller may overwrite it).  The all-to-all needs a dst: in place, storing segment
// p would overwrite what rank p is still reading.
template <class L, int OP, bool A2A>
__global__ void __launch_bounds__(kThreads) segments_pull_kernel(ARArgs a) {
  const int rank = a.rank, world = a.world;
  uint32_t epoch = barrier_epoch_load(a.sig, rank);
  const size_t seg = a.n_vec / world;
  const size_t stride = (size_t)gridDim.x * kThreads;
  const size_t first = (size_t)blockIdx.x * kThreads + threadIdx.x;
  uint4* mine = reinterpret_cast<uint4*>(a.bufs.p[rank]);
  if (a.src != nullptr) {
    for (int s = 0; s < world; ++s)
      for (size_t j = first; j < seg; j += stride)
        st_cg_v4(mine + (size_t)s * seg + j, ld_cg_v4(reinterpret_cast<const uint4*>(a.src) + (size_t)s * seg + j));
  }
  block_barrier_all_ranks(a.sig, rank, world, ++epoch);          // every rank's segments are in place
  const size_t off = (size_t)rank * seg;
  uint4* out = a.dst != nullptr ? reinterpret_cast<uint4*>(a.dst) : mine + off;
  for (size_t base = first; base < seg; base += stride * kUnroll) {
    uint4 raw[kUnroll][B2_MAX_RANKS];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const size_t j = base + (size_t)u * stride;
#pragma unroll
      for (int r = 0; r < B2_MAX_RANKS; ++r)
        if (r < world && j < seg) raw[u][r] = ld_cg_v4(reinterpret_cast<const uint4*>(a.bufs.p[r]) + off + j);
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const size_t j = base + (size_t)u * stride;
      if (j >= seg) continue;
      if constexpr (A2A) {
#pragma unroll
        for (int r = 0; r < B2_MAX_RANKS; ++r)
          if (r < world) st_cg_v4(out + (size_t)r * seg + j, raw[u][r]);
      } else {
        typename L::Acc acc[L::kElems];
        L::template zero<OP>(acc);
#pragma unroll
        for (int r = 0; r < B2_MAX_RANKS; ++r)
          if (r < world) L::template add<OP>(acc, raw[u][r]);
        st_cg_v4(out + j, L::template pack<OP>(acc, 1.f));
      }
    }
  }
  block_barrier_all_ranks(a.sig, rank, world, ++epoch);          // no peer reads this buffer any more
  if (threadIdx.x == 0) barrier_epoch_store(a.sig, rank, epoch);
}

// LL: vector v of segment d goes as flag-in-data lines to rank d's inbox, in the region of source `rank`, for every d != rank;
// then the W - 1 lines of this rank's own segment are awaited.  Reduce-scatter combines them with its own vector in rank order;
// all-to-all stores the line from source p at output segment p.  Per vector every rank pushes one line to every peer and waits
// for one from every peer, and vector v belongs to block v / kThreads, so the parity argument of allreduce_ll_kernel holds for
// any mix of calls on one inbox.  In place (no src / dst) the input is this rank's buffer and the reduce-scatter's output its
// segment `rank`; a thread reads every input vector it needs before it stores.
template <class L, int OP, bool A2A>
__global__ void __launch_bounds__(kThreads) segments_ll_kernel(ARArgs a) {
  const int rank = a.rank, world = a.world;
  const uint32_t epoch = barrier_epoch_load(a.sig, rank) + 1u;
  const uint32_t flag = epoch == 0u ? 1u : epoch;
  const size_t par = (size_t)(epoch & 1u);
  const size_t stride = (size_t)gridDim.x * kThreads;
  const size_t seg = a.n_vec / world;
  const uint4* in = reinterpret_cast<const uint4*>(a.src != nullptr ? a.src : a.bufs.p[rank]);
  uint4* out = a.dst != nullptr ? reinterpret_cast<uint4*>(a.dst) : reinterpret_cast<uint4*>(a.bufs.p[rank]) + (size_t)rank * seg;
  for (size_t v = (size_t)blockIdx.x * kThreads + threadIdx.x; v < seg; v += stride) {
    const size_t line = ((par * (size_t)world + (size_t)rank) * a.ll_cap + v) * 2;
#pragma unroll
    for (int i = 1; i < B2_MAX_RANKS; ++i) {
      if (i < world) {
        int d = rank + i;
        if (d >= world) d -= world;
        const uint4 w = ld_cg_v4(in + (size_t)d * seg + v);
        uint4* dl = reinterpret_cast<uint4*>(a.inbox.p[d]) + line;
        st_volatile_v4(dl, make_uint4(w.x, flag, w.y, flag));
        st_volatile_v4(dl + 1, make_uint4(w.z, flag, w.w, flag));
      }
    }
    const uint4 own = ld_cg_v4(in + (size_t)rank * seg + v);
    typename L::Acc acc[L::kElems];
    if constexpr (!A2A) L::template zero<OP>(acc);
    const uint4* box = reinterpret_cast<const uint4*>(a.inbox.p[rank]);
#pragma unroll
    for (int r = 0; r < B2_MAX_RANKS; ++r) {
      if (r < world) {
        uint4 w;
        if (r == rank) {
          w = own;
        } else {
          const uint4* src = box + ((par * (size_t)world + (size_t)r) * a.ll_cap + v) * 2;
          uint4 q0, q1;
          unsigned long long spins = 0;
          for (;;) {
            q0 = ld_volatile_v4(src);
            q1 = ld_volatile_v4(src + 1);
            if (q0.y == flag && q0.w == flag && q1.y == flag && q1.w == flag) break;
            if (++spins > B2_SPIN_LIMIT) {
              printf("[b200dist] LL %s: rank %d timed out waiting for rank %d (block %d, epoch %u)\n",
                     A2A ? "all-to-all" : "reduce-scatter", rank, r, (int)blockIdx.x, flag);
              __trap();
            }
          }
          w = make_uint4(q0.x, q0.z, q1.x, q1.z);
        }
        if constexpr (A2A) st_cg_v4(out + (size_t)r * seg + v, w);
        else L::template add<OP>(acc, w);                             // fixed rank order, as the all-reduce
      }
    }
    if constexpr (!A2A) st_cg_v4(out + v, L::template pack<OP>(acc, 1.f));
  }
  __syncthreads();
  if (threadIdx.x == 0) barrier_epoch_store(a.sig, rank, epoch);
}

// ------------------------------------------------------------------------------------------ all-to-allv
// Variable segments of raw bytes: rank r sends src[d] (src_bytes[d] bytes) to rank d and receives what rank p sends it into
// dst[p] (dst_bytes[p] bytes).  The staging buffer of every rank is [header | half 0 | half 1]: the header holds this rank's W
// send lengths, each half W slots of kA2avChunk bytes, slot d for what goes to rank d.  Neither its size nor the grid depends on
// the lengths, which ranks cannot agree on without communicating: segments move in rounds of at most kA2avChunk bytes per pair.
//
//   stage chunk 0 of every send into half 0, publish the header, barrier
//   every rank reads all W x W lengths: K = max(1, ceil(max / kA2avChunk)), the same on every rank
//   round k < K: pull chunk k of segment `rank` from every rank's half k & 1 into dst, stage chunk k + 1 into half (k + 1) & 1,
//                barrier
//
// K + 1 barriers in all.  Half h is staged again in round k + 1 only after the barrier that ends round k, the last round whose
// pulls read it, and the barrier that ends round K - 1 is the one after which no peer reads this buffer (header included), as
// segments_pull_kernel ends.  Vector j of every slot is staged and pulled by one (block, thread) in every round and on every
// rank, and every block writes the header itself (identical values), so the per-block barriers order everything a block
// reads.  The receiver moves min(what the sender published, what it expects) of each pair: splits that disagree between ranks
// give a truncated segment, never a write outside one or a different number of rounds.
constexpr size_t kA2avChunk = 128 << 10;     // bytes per (source, destination) pair and round: an unmeasured starting point
constexpr size_t kA2avHeader = 16 * ((B2_MAX_RANKS * 8 + 15) / 16);   // W 8-byte send lengths, 16-byte aligned
constexpr size_t kA2avChunkVec = kA2avChunk / 16;

struct A2AVArgs {
  PeerPtrs bufs;                                   // staging buffer of every rank: header | half 0 | half 1
  SignalPads sig;
  const unsigned char* src[B2_MAX_RANKS];          // what this rank sends to rank d ...
  unsigned long long src_bytes[B2_MAX_RANKS];      // ... and how many bytes
  unsigned char* dst[B2_MAX_RANKS];                // where what rank p sends lands ...
  unsigned long long dst_bytes[B2_MAX_RANKS];      // ... and how many bytes this rank expects from it
  int rank, world;
};

__device__ __forceinline__ void st_cg_u64(void* p, unsigned long long v) {
  asm volatile("st.global.cg.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_cg_u64(const void* p) {
  unsigned long long v;
  asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// The n (> 0) bytes of a segment at p, at most 16 of them, as one vector: a whole vector with the widest accesses p's alignment
// allows, a partial one byte by byte, so that no byte outside the segment is read.  The bytes past n are zero.
__device__ __forceinline__ uint4 a2av_load(const unsigned char* p, size_t n) {
  const uintptr_t at = reinterpret_cast<uintptr_t>(p);
  if (n >= 16) {
    if ((at & 15) == 0) return ld_cg_v4(p);
    if ((at & 7) == 0) {
      const uint2 x = reinterpret_cast<const uint2*>(p)[0], y = reinterpret_cast<const uint2*>(p)[1];
      return make_uint4(x.x, x.y, y.x, y.y);
    }
    if ((at & 3) == 0) {
      const uint32_t* q = reinterpret_cast<const uint32_t*>(p);
      return make_uint4(q[0], q[1], q[2], q[3]);
    }
  }
  uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
  for (int i = 0; i < 16; ++i)
    if ((size_t)i < n) w[i >> 2] |= (uint32_t)p[i] << (8 * (i & 3));
  return make_uint4(w[0], w[1], w[2], w[3]);
}

// Store the first n (> 0, at most 16 used) bytes of v at p, never a byte past p + n: a partial vector must not clobber what
// follows the segment.
__device__ __forceinline__ void a2av_store(unsigned char* p, size_t n, uint4 v) {
  const uintptr_t at = reinterpret_cast<uintptr_t>(p);
  if (n >= 16) {
    if ((at & 15) == 0) return st_cg_v4(p, v);
    if ((at & 7) == 0) {
      reinterpret_cast<uint2*>(p)[0] = make_uint2(v.x, v.y);
      reinterpret_cast<uint2*>(p)[1] = make_uint2(v.z, v.w);
      return;
    }
    if ((at & 3) == 0) {
      uint32_t* q = reinterpret_cast<uint32_t*>(p);
      q[0] = v.x; q[1] = v.y; q[2] = v.z; q[3] = v.w;
      return;
    }
  }
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 16; ++i)
    if ((size_t)i < n) p[i] = (unsigned char)(w[i >> 2] >> (8 * (i & 3)));
}

// Stage bytes [off, off + kA2avChunk) of every send into `half` of this rank's buffer (slot d for rank d).
__device__ __forceinline__ void a2av_stage(const A2AVArgs& a, unsigned char* half, size_t off, size_t first, size_t stride) {
  for (size_t j = first; j < kA2avChunkVec; j += stride) {
    const size_t at = off + j * 16;
#pragma unroll
    for (int d = 0; d < B2_MAX_RANKS; ++d)
      if (d < a.world && at < a.src_bytes[d])
        st_cg_v4(half + (size_t)d * kA2avChunk + j * 16, a2av_load(a.src[d] + at, a.src_bytes[d] - at));
  }
}

__global__ void __launch_bounds__(kThreads) alltoallv_kernel(A2AVArgs a) {
  const int rank = a.rank, world = a.world;
  uint32_t epoch = barrier_epoch_load(a.sig, rank);
  const size_t stride = (size_t)gridDim.x * kThreads;
  const size_t first = (size_t)blockIdx.x * kThreads + threadIdx.x;
  const size_t half_bytes = (size_t)world * kA2avChunk;
  unsigned char* mine = reinterpret_cast<unsigned char*>(a.bufs.p[rank]);
  __shared__ unsigned long long take_s[B2_MAX_RANKS];       // bytes this rank takes from rank s
  __shared__ unsigned long long longest;                    // the longest send of any rank
  if (threadIdx.x < (unsigned)world) st_cg_u64(mine + 8 * threadIdx.x, a.src_bytes[threadIdx.x]);
  if (threadIdx.x == 0) longest = 0;
  a2av_stage(a, mine + kA2avHeader, 0, first, stride);
  block_barrier_all_ranks(a.sig, rank, world, ++epoch);          // every header and chunk 0 are in place
  if (threadIdx.x < (unsigned)(world * world)) {
    const int s = threadIdx.x / world, d = threadIdx.x % world;
    const unsigned long long n = ld_cg_u64(reinterpret_cast<const unsigned char*>(a.bufs.p[s]) + 8 * d);
    atomicMax(&longest, n);
    if (d == rank) take_s[s] = n < a.dst_bytes[s] ? n : a.dst_bytes[s];
  }
  __syncthreads();
  unsigned long long take[B2_MAX_RANKS];
#pragma unroll
  for (int s = 0; s < B2_MAX_RANKS; ++s) take[s] = s < world ? take_s[s] : 0ull;
  const unsigned long long rounds = longest == 0 ? 1ull : (longest + kA2avChunk - 1) / kA2avChunk;
  for (unsigned long long k = 0; k < rounds; ++k) {
    const size_t off = (size_t)k * kA2avChunk;
    const size_t cur = kA2avHeader + (size_t)(k & 1) * half_bytes + (size_t)rank * kA2avChunk;
    for (size_t j = first; j < kA2avChunkVec; j += stride) {
      const size_t at = off + j * 16;
      uint4 raw[B2_MAX_RANKS];
#pragma unroll
      for (int s = 0; s < B2_MAX_RANKS; ++s)
        if (s < world && at < take[s]) raw[s] = ld_cg_v4(reinterpret_cast<const unsigned char*>(a.bufs.p[s]) + cur + j * 16);
#pragma unroll
      for (int s = 0; s < B2_MAX_RANKS; ++s)
        if (s < world && at < take[s]) a2av_store(a.dst[s] + at, take[s] - at, raw[s]);
    }
    if (k + 1 < rounds) a2av_stage(a, mine + kA2avHeader + (size_t)((k + 1) & 1) * half_bytes, off + kA2avChunk, first, stride);
    block_barrier_all_ranks(a.sig, rank, world, ++epoch);        // round k read; after the last, no peer reads this buffer
  }
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

template <class L, int OP, bool ROOT>
void launch_kernel(int variant, dim3 grid, const ARArgs& a, cudaStream_t stream) {
  if (variant == 0) allreduce_oneshot_kernel<L, OP, ROOT><<<grid, kThreads, 0, stream>>>(a);
  else if (variant == 1) allreduce_twoshot_kernel<L, false, OP, ROOT><<<grid, kThreads, 0, stream>>>(a);
  else if (variant == 3) allreduce_ll_kernel<L, OP, ROOT><<<grid, kThreads, 0, stream>>>(a);
  else if constexpr (OP == kSum && !ROOT && L::kNvls) allreduce_twoshot_kernel<L, true, kSum, false><<<grid, kThreads, 0, stream>>>(a);
}

template <class L, int OP>
void launch_lane(int variant, dim3 grid, const ARArgs& a, cudaStream_t stream) {
  if (a.root >= 0) launch_kernel<L, OP, true>(variant, grid, a, stream);
  else launch_kernel<L, OP, false>(variant, grid, a, stream);
}

template <int OP>
void launch_op(int variant, int dtype, dim3 grid, const ARArgs& a, cudaStream_t stream) {
  if constexpr (OP < kBcast) {
    switch (dtype) {
      case kBF16: return launch_lane<LaneBF16, OP>(variant, grid, a, stream);
      case kF16: return launch_lane<LaneF16, OP>(variant, grid, a, stream);
      case kF64: return launch_lane<LaneF64, OP>(variant, grid, a, stream);
      case kI32: return launch_lane<LaneI32, OP>(variant, grid, a, stream);
      case kI64: return launch_lane<LaneI64, OP>(variant, grid, a, stream);
      case kI8: return launch_lane<LaneI8<true>, OP>(variant, grid, a, stream);
      case kU8:
      case kBool:                             // SUM / PRODUCT wrap to the same bits for both signs: one instance
        if constexpr (OP == kSum || OP == kProd) return launch_lane<LaneI8<true>, OP>(variant, grid, a, stream);
        else return launch_lane<LaneI8<false>, OP>(variant, grid, a, stream);
      default: return launch_lane<LaneF32, OP>(variant, grid, a, stream);
    }
  }
  if constexpr (OP == kGather) {
    if (a.root >= 0) return launch_kernel<LaneF32, kGather, true>(variant, grid, a, stream);
  }
  launch_kernel<LaneF32, OP, false>(variant, grid, a, stream);
}

template <class L, int OP, bool A2A>
void launch_segments(int variant, dim3 grid, const ARArgs& a, cudaStream_t stream) {
  if (variant == 3) segments_ll_kernel<L, OP, A2A><<<grid, kThreads, 0, stream>>>(a);
  else segments_pull_kernel<L, OP, A2A><<<grid, kThreads, 0, stream>>>(a);
}

template <int OP>
void launch_reduce_scatter(int variant, int dtype, dim3 grid, const ARArgs& a, cudaStream_t stream) {
  switch (dtype) {
    case kBF16: return launch_segments<LaneBF16, OP, false>(variant, grid, a, stream);
    case kF16: return launch_segments<LaneF16, OP, false>(variant, grid, a, stream);
    case kF64: return launch_segments<LaneF64, OP, false>(variant, grid, a, stream);
    case kI32: return launch_segments<LaneI32, OP, false>(variant, grid, a, stream);
    case kI64: return launch_segments<LaneI64, OP, false>(variant, grid, a, stream);
    case kI8: return launch_segments<LaneI8<true>, OP, false>(variant, grid, a, stream);
    case kU8:
    case kBool:                               // as launch_op: SUM / PRODUCT share the int8 instance
      if constexpr (OP == kSum || OP == kProd) return launch_segments<LaneI8<true>, OP, false>(variant, grid, a, stream);
      else return launch_segments<LaneI8<false>, OP, false>(variant, grid, a, stream);
    default: return launch_segments<LaneF32, OP, false>(variant, grid, a, stream);
  }
}

// The grid of a reduce-scatter or all-to-all: one thread per vector of a segment.  LL: sized by the segment alone (<= ll_cap),
// never by max_blocks, so vector v belongs to block v / kThreads as in every LL call on the inbox.
inline dim3 segments_grid(int variant, size_t seg, int max_blocks) {
  if (max_blocks <= 0 || max_blocks > B2_MAX_BLOCKS) max_blocks = B2_MAX_BLOCKS;
  size_t blocks = (seg + kThreads - 1) / kThreads;
  if (blocks < 1) blocks = 1;
  const size_t cap = variant == 3 ? (size_t)B2_MAX_BLOCKS : (size_t)max_blocks;
  return dim3((unsigned)(blocks > cap ? cap : blocks));
}

// Shared checks and arguments of the two segmented launchers; false for a call they refuse.
inline bool segments_args(int variant, const PeerPtrs* bufs, const SignalPads* sig, const void* src, void* dst, size_t n_vec,
                          int rank, int world, const PeerPtrs* inbox, size_t ll_cap, ARArgs* a) {
  if ((variant != 0 && variant != 3) || world < 1 || world > B2_MAX_RANKS || rank < 0 || rank >= world) return false;
  if (bufs == nullptr || sig == nullptr || n_vec % (size_t)world != 0) return false;
  memset(a, 0, sizeof(*a));
  a->bufs = *bufs; a->sig = *sig; a->src = src; a->dst = dst; a->n_vec = n_vec; a->scale = 1.f;
  a->rank = rank; a->world = world; a->root = -1;
  if (variant == 3) {
    if (inbox == nullptr || ll_cap < n_vec / world) return false;
    a->inbox = *inbox;
    a->ll_cap = ll_cap;
  }
  return true;
}

}  // namespace b2

// ============================================================================================ launchers
extern "C" {

// variant: 0 one-shot, 1 two-shot, 2 NVLS, 3 LL (needs inbox / ll_cap).  op: 0 SUM, 1 PRODUCT, 2 MAX, 3 MIN, 4 broadcast
// from `root`, 5 all-gather, or with root >= 0 gather to `root`, 6 scatter from `root`; a reduction with root >= 0 is a
// reduce to that rank.  dtype: the wire dtype of a reduction, 0 fp32, 1 bf16 (the locals may be fp32 for SUM), 2 fp16,
// 3 fp64, 4 int8, 5 uint8, 6 int32, 7 int64, 8 bool (the uint8 ops; the caller maps a bool SUM to MAX); 0 for the raw moves.
// Returns cudaError_t as int; cudaErrorInvalidValue, without a launch, for an unknown variant, op or dtype, a world outside
// 1..8, a rank outside [0, world), a root outside [-1, world) (a broadcast and a scatter need one), a scale other than 1,
// fp32 locals over a bf16 wire or NVLS for any op but SUM, a scale, fp32 locals or NVLS for any dtype but fp32 / bf16, a bool
// SUM, a dtype other than 0 for the raw moves, a two-shot / NVLS / gather / scatter n_vec that is not a multiple of world (the
// remainder would be left out) or an LL message larger than the inbox.
int b2_allreduce_dtype_launch(int variant, int dtype, const PeerPtrs* bufs, const b2::SignalPads* sig, void* mc,
                              const void* src, int src_f32, void* dst, int dst_f32, size_t n_vec, float scale,
                              int rank, int world, int max_blocks, const PeerPtrs* inbox, size_t ll_cap, int op, int root,
                              cudaStream_t stream) {
  if (variant < 0 || variant > 3 || world < 1 || world > B2_MAX_RANKS || rank < 0 || rank >= world)
    return (int)cudaErrorInvalidValue;
  if (op < b2::kSum || op > b2::kScatter || root < -1 || root >= world) return (int)cudaErrorInvalidValue;
  if (dtype < b2::kF32 || dtype > b2::kBool) return (int)cudaErrorInvalidValue;
  if ((op == b2::kBcast || op == b2::kScatter) && root < 0) return (int)cudaErrorInvalidValue;
  if (op != b2::kSum && (scale != 1.f || src_f32 || dst_f32)) return (int)cudaErrorInvalidValue;
  if (variant == 2 && (op != b2::kSum || root >= 0)) return (int)cudaErrorInvalidValue;   // NVLS: the SUM all-reduce only
  if (op >= b2::kBcast && dtype != b2::kF32) return (int)cudaErrorInvalidValue;
  if (dtype >= b2::kF16 && (scale != 1.f || src_f32 || dst_f32 || variant == 2)) return (int)cudaErrorInvalidValue;
  if (dtype == b2::kBool && op == b2::kSum) return (int)cudaErrorInvalidValue;
  const bool segmented = op == b2::kGather || op == b2::kScatter;          // one segment of n_vec / world per rank
  if ((variant == 1 || variant == 2 || segmented) && n_vec % (size_t)world != 0)
    return (int)cudaErrorInvalidValue;                                     // slice = n_vec / world
  const size_t n_push = segmented ? n_vec / world : n_vec;                // LL: vectors each rank pushes
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
  const size_t work = variant == 0 ? (op == b2::kScatter ? n_push : n_vec) : variant == 3 ? n_push : n_vec / world;
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
    case b2::kSum: b2::launch_op<b2::kSum>(variant, dtype, grid, a, stream); break;
    case b2::kProd: b2::launch_op<b2::kProd>(variant, dtype, grid, a, stream); break;
    case b2::kMax: b2::launch_op<b2::kMax>(variant, dtype, grid, a, stream); break;
    case b2::kMin: b2::launch_op<b2::kMin>(variant, dtype, grid, a, stream); break;
    case b2::kBcast: b2::launch_op<b2::kBcast>(variant, dtype, grid, a, stream); break;
    case b2::kGather: b2::launch_op<b2::kGather>(variant, dtype, grid, a, stream); break;
    default: b2::launch_op<b2::kScatter>(variant, dtype, grid, a, stream); break;
  }
  return (int)cudaGetLastError();
}

// The fp32 / bf16 launcher of the collectives before the dtype code: `bf16` selects the bf16 wire.
int b2_allreduce_launch(int variant, int bf16, const PeerPtrs* bufs, const b2::SignalPads* sig, void* mc,
                        const void* src, int src_f32, void* dst, int dst_f32, size_t n_vec, float scale,
                        int rank, int world, int max_blocks, const PeerPtrs* inbox, size_t ll_cap, int op, int root,
                        cudaStream_t stream) {
  return b2_allreduce_dtype_launch(variant, bf16 ? b2::kBF16 : b2::kF32, bufs, sig, mc, src, src_f32, dst, dst_f32, n_vec,
                                   scale, rank, world, max_blocks, inbox, ll_cap, op, root, stream);
}

// Reduce-scatter: n_vec 16-byte vectors of input on every rank, world segments of n_vec / world; rank r's output (dst, or
// with dst null segment r of its own buffer) is segment r of the reduction.  src null: the input already is the buffer.
// variant 0 pull (barriers), 3 LL (needs inbox / ll_cap).  op and dtype as b2_allreduce_dtype_launch (wire dtype = local
// dtype, no scale; a bool SUM is refused, the caller maps it to MAX).  Returns cudaError_t as int; cudaErrorInvalidValue,
// without a launch, for a variant other than 0 / 3, an unknown op or dtype, a bool SUM, a world outside 1..8, a rank outside
// [0, world), an n_vec that is not a multiple of world, or an LL segment larger than the inbox.
int b2_reduce_scatter_launch(int variant, int dtype, int op, const PeerPtrs* bufs, const b2::SignalPads* sig, const void* src,
                             void* dst, size_t n_vec, int rank, int world, int max_blocks, const PeerPtrs* inbox,
                             size_t ll_cap, cudaStream_t stream) {
  if (op < b2::kSum || op > b2::kMin || dtype < b2::kF32 || dtype > b2::kBool) return (int)cudaErrorInvalidValue;
  if (dtype == b2::kBool && op == b2::kSum) return (int)cudaErrorInvalidValue;
  b2::ARArgs a;
  if (!b2::segments_args(variant, bufs, sig, src, dst, n_vec, rank, world, inbox, ll_cap, &a)) return (int)cudaErrorInvalidValue;
  const dim3 grid = b2::segments_grid(variant, n_vec / world, max_blocks);
  switch (op) {
    case b2::kSum: b2::launch_reduce_scatter<b2::kSum>(variant, dtype, grid, a, stream); break;
    case b2::kProd: b2::launch_reduce_scatter<b2::kProd>(variant, dtype, grid, a, stream); break;
    case b2::kMax: b2::launch_reduce_scatter<b2::kMax>(variant, dtype, grid, a, stream); break;
    default: b2::launch_reduce_scatter<b2::kMin>(variant, dtype, grid, a, stream); break;
  }
  return (int)cudaGetLastError();
}

// All-to-all of raw 16-byte vectors: segment p of rank r's dst receives segment r of rank p's input (src, or with src null
// this rank's buffer).  dst is required: an in-place all-to-all would overwrite segments its peers are still reading.
// Refusals as b2_reduce_scatter_launch, plus a null dst.
int b2_alltoall_launch(int variant, const PeerPtrs* bufs, const b2::SignalPads* sig, const void* src, void* dst, size_t n_vec,
                       int rank, int world, int max_blocks, const PeerPtrs* inbox, size_t ll_cap, cudaStream_t stream) {
  if (dst == nullptr) return (int)cudaErrorInvalidValue;
  b2::ARArgs a;
  if (!b2::segments_args(variant, bufs, sig, src, dst, n_vec, rank, world, inbox, ll_cap, &a)) return (int)cudaErrorInvalidValue;
  b2::launch_segments<b2::LaneF32, b2::kSum, true>(variant, b2::segments_grid(variant, n_vec / world, max_blocks), a, stream);
  return (int)cudaGetLastError();
}

// The staging layout of the all-to-allv: kA2avChunk bytes per pair and round behind a header of `header` bytes, so a world
// of W ranks needs header + 2 x W x chunk bytes of symmetric buffer.
void b2_alltoallv_config(size_t* chunk, size_t* header) {
  *chunk = b2::kA2avChunk;
  *header = b2::kA2avHeader;
}

// All-to-allv of raw bytes (alltoallv_kernel): src[d] / src_bytes[d] is what this rank sends to rank d, dst[p] / dst_bytes[p]
// where what rank p sends lands; bufs are staging buffers of at least header + 2 x world x chunk bytes (b2_alltoallv_config).
// The grid is min(chunk / 16 / kThreads, max_blocks) on every rank, whatever the lengths.  Returns cudaError_t as int;
// cudaErrorInvalidValue, without a launch, for a world outside 1..8, a rank outside [0, world), or a null pointer with a
// non-zero byte count.
int b2_alltoallv_launch(const PeerPtrs* bufs, const b2::SignalPads* sig, const void* const* src, const unsigned long long* src_bytes,
                        void* const* dst, const unsigned long long* dst_bytes, int rank, int world, int max_blocks,
                        cudaStream_t stream) {
  if (world < 1 || world > B2_MAX_RANKS || rank < 0 || rank >= world || bufs == nullptr || sig == nullptr)
    return (int)cudaErrorInvalidValue;
  b2::A2AVArgs a;
  memset(&a, 0, sizeof(a));
  a.bufs = *bufs; a.sig = *sig; a.rank = rank; a.world = world;
  for (int r = 0; r < world; ++r) {
    if (bufs->p[r] == nullptr || (src_bytes[r] != 0 && src[r] == nullptr) || (dst_bytes[r] != 0 && dst[r] == nullptr))
      return (int)cudaErrorInvalidValue;
    a.src[r] = static_cast<const unsigned char*>(src[r]); a.src_bytes[r] = src_bytes[r];
    a.dst[r] = static_cast<unsigned char*>(dst[r]); a.dst_bytes[r] = dst_bytes[r];
  }
  if (max_blocks <= 0 || max_blocks > B2_MAX_BLOCKS) max_blocks = B2_MAX_BLOCKS;
  size_t blocks = (b2::kA2avChunkVec + b2::kThreads - 1) / b2::kThreads;
  if (blocks > (size_t)max_blocks) blocks = (size_t)max_blocks;
  b2::alltoallv_kernel<<<dim3((unsigned)blocks), b2::kThreads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

int b2_barrier_launch(const b2::SignalPads* sig, int rank, int world, cudaStream_t stream) {
  b2::barrier_kernel<<<1, 32, 0, stream>>>(*sig, rank, world);
  return (int)cudaGetLastError();
}

}  // extern "C"
