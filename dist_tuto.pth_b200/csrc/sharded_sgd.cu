// Sharded optimizer step for generic models on sm_90a: reduce-scatter of one gradient bucket, momentum SGD on the slice this
// rank owns and all-gather of the updated PARAMETERS, in one launch per bucket.
//
// The two-shot all-reduce (allreduce.cu) has rank r reduce slice r and push the averaged gradient slice to every rank, where a
// second kernel (sgd_flat_kernel, sgd.cu) then applies the same update W times over.  Here the owner of slice r applies the
// update itself and pushes the new parameters instead: the NVLink bytes are the same, the second kernel is gone, and the
// momentum exists for the owned slice only (optimizer state is 1/W per GPU).
//
// Same grid and slice mapping as allreduce_twoshot_kernel: slice = n_vec / world, rank r owns vectors [r*slice, (r+1)*slice)
// of the gradient bucket, and vector j of a slice belongs to the same (block, thread) on every rank and in every phase, so
// the per-block barriers order everything a block touches.
//
//   barrier                      every rank's gradients of this bucket are complete
//   owned slice, per vector      g = (((0 + g_0) + g_1) + ...) * scale in fp32, in rank order (bit for bit what the one-shot and
//                                two-shot all-reduce store for an fp32 bucket); sgd_flat_kernel's fmaf sequence on the own
//                                parameter and momentum vectors; momentum stored locally; the new parameter vector stored
//                                into EVERY rank's parameter flat
//   barrier                      every parameter slice has landed everywhere, and every peer has finished reading this rank's
//                                gradients
//   zero the local bucket        only now: before that barrier the peers are still loading this bucket's slices
//
// A bf16 bucket (8 gradients per vector) updates two fp32 parameter vectors per gradient vector.  The fp32 sum x scale feeds
// the update unrounded: the averaged gradient never takes a bf16 round trip.
//
// The update is a template parameter of the one kernel (sharded_step_kernel): ShardedSgdUpdate (momentum SGD, FlatSGD) and
// ShardedAdamwUpdate (AdamW, FlatAdamW: adamw_elem of adamw_device.cuh on the slice's first and second moment shards).  An
// update type names its argument struct, which carries the fields the skeleton reads (grads, params, sig, n_vec, scale, rank,
// world, zero_grad), loads its optimizer state for a parameter vector, applies the update and stores the state back.
//
// With parameter groups, ShardedSgdGroupedUpdate and ShardedAdamwGroupedUpdate load a group id next to the state of each
// parameter vector and take that group's scalars; the skeleton and the other instances are unchanged.
//
// Capturable<U> (FlatSGD / FlatAdamW capturable=True, flat_scalars.cuh) is U with its scalars read from the device scalar
// block: the skeleton calls its begin() once per CTA, which copies them to shared memory; the other instances compile
// without that call.
//
// ShardedRmspropUpdate and ShardedRmspropGroupedUpdate (FlatRMSprop) are two more update types of the same skeleton:
// rmsprop_elem of rmsprop_device.cuh on the slice's square-average shard and, when the update has them, its momentum and
// centered-average shards.  Capturable<U> takes their lr and weight decay from the block, the other scalars from the
// arguments.
#include <cstring>
#include <type_traits>
#include "adamw_device.cuh"
#include "common.cuh"
#include "flat_scalars.cuh"
#include "param_groups.cuh"
#include "rmsprop_device.cuh"
#include "shard_grid.h"

namespace b2 {

constexpr int kShardThreads = 512;   // as the all-reduce kernels (kThreads)
constexpr int kShardUnroll = 2;      // gradient vectors per thread and pass: 2 x world 16-byte peer loads in flight

struct ShardedSgdArgs {
  PeerPtrs grads;         // symmetric gradient bucket of every rank
  PeerPtrs params;        // symmetric fp32 parameter flat of every rank
  SignalPads sig;         // signal pad of the gradient bucket
  float* momentum;        // this rank's shard: the fp32 momentum of its slice only
  size_t n_vec;           // 16-byte vectors of the gradient bucket, a multiple of world
  float lr, mu, wd, scale;
  int rank, world, zero_grad;
};

struct ShardedAdamwArgs {
  PeerPtrs grads;         // as ShardedSgdArgs
  PeerPtrs params;
  SignalPads sig;
  float* exp_avg;         // this rank's shards of the first and second moments (its slice only)
  float* exp_avg_sq;
  size_t n_vec;
  AdamwScalars s;
  float scale;
  int rank, world, zero_grad;
};

// With parameter groups (FlatSGD / FlatAdamW param_groups): the same fields, plus this rank's group map (one uint8 id per
// fp32 parameter vector of its slice, kP x slice ids) and the per-group scalars (param_groups.cuh).
struct ShardedSgdGroupedArgs {
  PeerPtrs grads;
  PeerPtrs params;
  SignalPads sig;
  float* momentum;
  const uint8_t* map;
  size_t n_vec;
  float mu, scale;
  int rank, world, zero_grad;
  SgdGroups gs;
};

struct ShardedAdamwGroupedArgs {
  PeerPtrs grads;
  PeerPtrs params;
  SignalPads sig;
  float* exp_avg;
  float* exp_avg_sq;
  const uint8_t* map;
  size_t n_vec;
  AdamwScalars s;         // decay and step_size unused: they come from the vector's group
  float scale;
  int rank, world, zero_grad;
  AdamwGroups gs;
};

// FlatRMSprop: this rank's shards of the square average and, when they exist (s.centered / s.momentum), of the centered
// gradient average and the momentum buffer; null otherwise.  Grouped: `s` without lr / wd, which come from the vector's group.
struct ShardedRmspropArgs {
  PeerPtrs grads;
  PeerPtrs params;
  SignalPads sig;
  float* square_avg;
  float* grad_avg;
  float* momentum_buffer;
  size_t n_vec;
  RmspropScalars s;
  float scale;
  int rank, world, zero_grad;
};

struct ShardedRmspropGroupedArgs {
  PeerPtrs grads;
  PeerPtrs params;
  SignalPads sig;
  float* square_avg;
  float* grad_avg;
  float* momentum_buffer;
  const uint8_t* map;
  size_t n_vec;
  RmspropScalars s;
  float scale;
  int rank, world, zero_grad;
  SgdGroups gs;
};

// The per-vector updates of sharded_step_kernel.  q indexes the fp32 state vector within this rank's shard.
template <bool kNesterov>
struct ShardedSgdUpdate {
  using Args = ShardedSgdArgs;
  static constexpr int kUnroll = kShardUnroll;
  float4 m;
  __device__ __forceinline__ void load(const Args& a, size_t q) { m = reinterpret_cast<float4*>(a.momentum)[q]; }
  __device__ __forceinline__ void apply(const Args& a, float4& p, float4 g) { sgd4<kNesterov>(p, m, g, a.lr, a.mu, a.wd); }
  __device__ __forceinline__ void store(const Args& a, size_t q) { reinterpret_cast<float4*>(a.momentum)[q] = m; }
};

struct ShardedAdamwUpdate {
  using Args = ShardedAdamwArgs;
  static constexpr int kUnroll = 1;       // two moment vectors per parameter vector: unroll 2 would not fit in 128 registers
  float4 m, v;
  __device__ __forceinline__ void load(const Args& a, size_t q) {
    m = reinterpret_cast<float4*>(a.exp_avg)[q];
    v = reinterpret_cast<float4*>(a.exp_avg_sq)[q];
  }
  __device__ __forceinline__ void apply(const Args& a, float4& p, float4 g) { adamw4(p, m, v, g, a.s); }
  __device__ __forceinline__ void store(const Args& a, size_t q) {
    reinterpret_cast<float4*>(a.exp_avg)[q] = m;
    reinterpret_cast<float4*>(a.exp_avg_sq)[q] = v;
  }
};

// Grouped instances: the group id of the vector is loaded next to its state, and the update takes that group's scalars.
template <bool kNesterov>
struct ShardedSgdGroupedUpdate {
  using Args = ShardedSgdGroupedArgs;
  static constexpr int kUnroll = kShardUnroll;
  float4 m;
  int gid;
  __device__ __forceinline__ void load(const Args& a, size_t q) {
    m = reinterpret_cast<float4*>(a.momentum)[q];
    gid = a.map[q];
  }
  __device__ __forceinline__ void apply(const Args& a, float4& p, float4 g) {
    sgd4<kNesterov>(p, m, g, a.gs.lr[gid], a.mu, a.gs.wd[gid]);
  }
  __device__ __forceinline__ void store(const Args& a, size_t q) { reinterpret_cast<float4*>(a.momentum)[q] = m; }
};

struct ShardedAdamwGroupedUpdate {
  using Args = ShardedAdamwGroupedArgs;
  static constexpr int kUnroll = 1;
  float4 m, v;
  int gid;
  __device__ __forceinline__ void load(const Args& a, size_t q) {
    m = reinterpret_cast<float4*>(a.exp_avg)[q];
    v = reinterpret_cast<float4*>(a.exp_avg_sq)[q];
    gid = a.map[q];
  }
  __device__ __forceinline__ void apply(const Args& a, float4& p, float4 g) {
    AdamwScalars s = a.s;
    s.decay = a.gs.decay[gid];
    s.step_size = a.gs.step_size[gid];
    adamw4(p, m, v, g, s);
  }
  __device__ __forceinline__ void store(const Args& a, size_t q) {
    reinterpret_cast<float4*>(a.exp_avg)[q] = m;
    reinterpret_cast<float4*>(a.exp_avg_sq)[q] = v;
  }
};

// RMSprop: up to three state vectors per parameter vector, so one gradient vector per thread and pass as for AdamW.  The
// absent states are neither loaded nor stored (uniform branches on s.centered / s.momentum).
template <class A>
__device__ __forceinline__ void rmsprop_load(const A& a, size_t q, float4& sq, float4& ga, float4& buf) {
  sq = reinterpret_cast<float4*>(a.square_avg)[q];
  if (a.s.centered) ga = reinterpret_cast<float4*>(a.grad_avg)[q];
  if (a.s.momentum) buf = reinterpret_cast<float4*>(a.momentum_buffer)[q];
}
template <class A>
__device__ __forceinline__ void rmsprop_store(const A& a, size_t q, float4 sq, float4 ga, float4 buf) {
  reinterpret_cast<float4*>(a.square_avg)[q] = sq;
  if (a.s.centered) reinterpret_cast<float4*>(a.grad_avg)[q] = ga;
  if (a.s.momentum) reinterpret_cast<float4*>(a.momentum_buffer)[q] = buf;
}

struct ShardedRmspropUpdate {
  using Args = ShardedRmspropArgs;
  static constexpr int kUnroll = 1;
  float4 sq, ga, buf;
  __device__ __forceinline__ void load(const Args& a, size_t q) { rmsprop_load(a, q, sq, ga, buf); }
  __device__ __forceinline__ void apply(const Args& a, float4& p, float4 g) { rmsprop4(p, sq, ga, buf, g, a.s); }
  __device__ __forceinline__ void store(const Args& a, size_t q) { rmsprop_store(a, q, sq, ga, buf); }
};

struct ShardedRmspropGroupedUpdate {
  using Args = ShardedRmspropGroupedArgs;
  static constexpr int kUnroll = 1;
  float4 sq, ga, buf;
  int gid;
  __device__ __forceinline__ void load(const Args& a, size_t q) {
    rmsprop_load(a, q, sq, ga, buf);
    gid = a.map[q];
  }
  __device__ __forceinline__ void apply(const Args& a, float4& p, float4 g) {
    RmspropScalars s = a.s;
    s.lr = a.gs.lr[gid];
    s.wd = a.gs.wd[gid];
    rmsprop4(p, sq, ga, buf, g, s);
  }
  __device__ __forceinline__ void store(const Args& a, size_t q) { rmsprop_store(a, q, sq, ga, buf); }
};

// Capturable instances (flat_scalars.cuh): Capturable<U> is the update U with the scalars its apply() reads taken from the
// scalar block on the device instead of the kernel arguments.  Its begin(), which the skeleton calls once per CTA, copies them
// into a shared copy of U's arguments; load(), apply() and store() are U's, apply() reading that copy.
__device__ __forceinline__ void cap_fill(ShardedSgdArgs& s, const ShardedSgdArgs& a, const FlatScalars& b) {
  if (threadIdx.x == 0) { s.lr = b.lr; s.wd = b.wd; s.mu = a.mu; }
}
__device__ __forceinline__ void cap_fill(ShardedAdamwArgs& s, const ShardedAdamwArgs&, const FlatScalars& b) {
  flat_block_load(s.s, b.adamw);
}
__device__ __forceinline__ void cap_fill(ShardedSgdGroupedArgs& s, const ShardedSgdGroupedArgs& a, const FlatScalars& b) {
  flat_block_load(s.gs, b.sgd);
  if (threadIdx.x == 0) s.mu = a.mu;
}
__device__ __forceinline__ void cap_fill(ShardedAdamwGroupedArgs& s, const ShardedAdamwGroupedArgs&, const FlatScalars& b) {
  flat_block_load(s.s, b.adamw);
  flat_block_load(s.gs, b.adamw_groups);
}

__device__ __forceinline__ void cap_fill(ShardedRmspropArgs& s, const ShardedRmspropArgs& a, const FlatScalars& b) {
  if (threadIdx.x == 0) { s.s = a.s; s.s.lr = b.lr; s.s.wd = b.wd; }
}
__device__ __forceinline__ void cap_fill(ShardedRmspropGroupedArgs& s, const ShardedRmspropGroupedArgs& a, const FlatScalars& b) {
  flat_block_load(s.gs, b.sgd);
  if (threadIdx.x == 0) s.s = a.s;
}

template <class A>
struct CapArgs : A {
  const FlatScalars* blk;
};

template <class U>
struct Capturable {
  using Args = CapArgs<typename U::Args>;
  static constexpr int kUnroll = U::kUnroll;
  U u;
  static __device__ __forceinline__ typename U::Args& scalars() {
    __shared__ typename U::Args s;
    return s;
  }
  static __device__ __forceinline__ void begin(const Args& a) {
    cap_fill(scalars(), a, *a.blk);
    __syncthreads();
  }
  __device__ __forceinline__ void load(const Args& a, size_t q) { u.load(a, q); }
  __device__ __forceinline__ void apply(const Args&, float4& p, float4 g) { u.apply(scalars(), p, g); }
  __device__ __forceinline__ void store(const Args& a, size_t q) { u.store(a, q); }
};

// Does the update have a per-CTA begin() (the capturable ones)?  The other instances compile without the call.
template <class U, class = void>
struct HasBegin : std::false_type {};
template <class U>
struct HasBegin<U, std::void_t<decltype(&U::begin)>> : std::true_type {};

__device__ __forceinline__ float4 as_f4(uint4 v) {
  return make_float4(__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z), __uint_as_float(v.w));
}
__device__ __forceinline__ uint4 as_u4(float4 v) {
  return make_uint4(__float_as_uint(v.x), __float_as_uint(v.y), __float_as_uint(v.z), __float_as_uint(v.w));
}

// kBf16: the gradient bucket is bf16 (8 elements per vector), else fp32 (4).  Parameters and optimizer state are fp32 in both.
template <bool kBf16, class Update>
__global__ void __launch_bounds__(kShardThreads) sharded_step_kernel(typename Update::Args a) {
  constexpr int kP = kBf16 ? 2 : 1;                     // fp32 parameter vectors per gradient vector
  constexpr int kUnroll = Update::kUnroll;           // gradient vectors per thread and pass
  if constexpr (HasBegin<Update>::value) Update::begin(a);
  const int rank = a.rank, world = a.world;
  uint32_t epoch = barrier_epoch_load(a.sig, rank);
  const size_t slice = a.n_vec / world;
  const size_t stride = (size_t)gridDim.x * kShardThreads;
  const size_t first = (size_t)blockIdx.x * kShardThreads + threadIdx.x;
  const size_t off = (size_t)rank * slice;
  const uint4* own = reinterpret_cast<const uint4*>(a.params.p[rank]) + kP * off;
  block_barrier_all_ranks(a.sig, rank, world, ++epoch);          // every rank's gradients are complete
  for (size_t base = first; base < slice; base += stride * kUnroll) {
    uint4 raw[kUnroll][B2_MAX_RANKS];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const size_t j = base + (size_t)u * stride;
#pragma unroll
      for (int r = 0; r < B2_MAX_RANKS; ++r)
        if (r < world && j < slice) raw[u][r] = ld_cg_v4(reinterpret_cast<const uint4*>(a.grads.p[r]) + off + j);
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const size_t j = base + (size_t)u * stride;
      if (j >= slice) continue;
      float4 p[kP], g[kP];
      Update st[kP];
#pragma unroll
      for (int h = 0; h < kP; ++h) {
        p[h] = as_f4(ld_cg_v4(own + kP * j + h));
        st[h].load(a, kP * j + h);
        g[h] = make_float4(0.f, 0.f, 0.f, 0.f);                  // the all-reduce's accumulator starts at +0 too
      }
#pragma unroll
      for (int r = 0; r < B2_MAX_RANKS; ++r) {
        if (r < world) {
          const uint4 v = raw[u][r];
          if constexpr (kBf16) {
            g[0].x += bf16lo(v.x); g[0].y += bf16hi(v.x); g[0].z += bf16lo(v.y); g[0].w += bf16hi(v.y);
            g[1].x += bf16lo(v.z); g[1].y += bf16hi(v.z); g[1].z += bf16lo(v.w); g[1].w += bf16hi(v.w);
          } else {
            g[0].x += __uint_as_float(v.x); g[0].y += __uint_as_float(v.y);
            g[0].z += __uint_as_float(v.z); g[0].w += __uint_as_float(v.w);
          }
        }
      }
#pragma unroll
      for (int h = 0; h < kP; ++h) {
        g[h].x *= a.scale; g[h].y *= a.scale; g[h].z *= a.scale; g[h].w *= a.scale;
        st[h].apply(a, p[h], g[h]);
        st[h].store(a, kP * j + h);
      }
#pragma unroll
      for (int r = 0; r < B2_MAX_RANKS; ++r) {
        if (r < world) {
#pragma unroll
          for (int h = 0; h < kP; ++h) st_cg_v4(reinterpret_cast<uint4*>(a.params.p[r]) + kP * (off + j) + h, as_u4(p[h]));
        }
      }
    }
  }
  // every parameter slice has landed everywhere; no peer reads this rank's gradients any more
  block_barrier_all_ranks(a.sig, rank, world, ++epoch);
  if (a.zero_grad) {
    uint4* mine = reinterpret_cast<uint4*>(a.grads.p[rank]);
    for (int s = 0; s < world; ++s)                               // vector j of every slice: the peers' block of the same index read it
      for (size_t j = first; j < slice; j += stride) mine[(size_t)s * slice + j] = make_uint4(0u, 0u, 0u, 0u);
  }
  if (threadIdx.x == 0) barrier_epoch_store(a.sig, rank, epoch);
}

}  // namespace b2

namespace {

// The checks of both launchers: cudaErrorInvalidValue (and no launch) for a world outside 1..8, a rank outside [0, world), an
// n_vec that is not a multiple of world (the remainder would be left out) or a null pointer.
bool shard_args_ok(const PeerPtrs* grads, const PeerPtrs* params, const b2::SignalPads* sig, size_t n_vec, int rank, int world) {
  if (world < 1 || world > B2_MAX_RANKS || rank < 0 || rank >= world) return false;
  if (grads == nullptr || params == nullptr || sig == nullptr) return false;
  if (n_vec % (size_t)world != 0) return false;
  for (int r = 0; r < world; ++r)
    if (grads->p[r] == nullptr || params->p[r] == nullptr || sig->pad[r] == nullptr) return false;
  return true;
}

static_assert(b2::kShardThreads == 512, "shard_grid.h sizes the grid for 512-thread CTAs");

}  // namespace

extern "C" {

// One sharded optimizer step of one bucket on `stream`.  n_vec: 16-byte vectors of the gradient bucket (4 fp32 or, with bf16,
// 8 bf16 gradients each); the parameter flats hold n_vec x 4 (x 8) floats and `momentum` n_vec / world x 4 (x 8).  The grid is
// the two-shot all-reduce's: ceil(ceil(slice / 512) / 2) CTAs, at most max_blocks.  Returns cudaError_t as int;
// cudaErrorInvalidValue, without a launch, for a world outside 1..8, a rank outside [0, world), an n_vec that is not a
// multiple of world (the remainder would be left out) or a null pointer.
int b2_sharded_sgd_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const b2::SignalPads* sig, float* momentum,
                          size_t n_vec, float lr, float mu, float wd, int nesterov, float scale, int zero_grad, int rank,
                          int world, int max_blocks, cudaStream_t stream) {
  if (momentum == nullptr || !shard_args_ok(grads, params, sig, n_vec, rank, world)) return (int)cudaErrorInvalidValue;
  b2::ShardedSgdArgs a;
  memset(&a, 0, sizeof(a));
  a.grads = *grads; a.params = *params; a.sig = *sig; a.momentum = momentum; a.n_vec = n_vec;
  a.lr = lr; a.mu = mu; a.wd = wd; a.scale = scale; a.rank = rank; a.world = world; a.zero_grad = zero_grad;
  const dim3 grid = shard_grid(n_vec, world, max_blocks);
  using namespace b2;
  if (bf16) {
    if (nesterov) sharded_step_kernel<true, ShardedSgdUpdate<true>><<<grid, kShardThreads, 0, stream>>>(a);
    else sharded_step_kernel<true, ShardedSgdUpdate<false>><<<grid, kShardThreads, 0, stream>>>(a);
  } else {
    if (nesterov) sharded_step_kernel<false, ShardedSgdUpdate<true>><<<grid, kShardThreads, 0, stream>>>(a);
    else sharded_step_kernel<false, ShardedSgdUpdate<false>><<<grid, kShardThreads, 0, stream>>>(a);
  }
  return (int)cudaGetLastError();
}

// The same step with AdamW (FlatAdamW): `exp_avg` and `exp_avg_sq` are this rank's moment shards, n_vec / world x 4 (x 8)
// floats each, and `s` the update's scalars (adamw_device.cuh).  Same grid, same refusals.
int b2_sharded_adamw_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const b2::SignalPads* sig, float* exp_avg,
                            float* exp_avg_sq, size_t n_vec, const b2::AdamwScalars* s, float scale, int zero_grad, int rank,
                            int world, int max_blocks, cudaStream_t stream) {
  if (exp_avg == nullptr || exp_avg_sq == nullptr || s == nullptr || !shard_args_ok(grads, params, sig, n_vec, rank, world))
    return (int)cudaErrorInvalidValue;
  b2::ShardedAdamwArgs a;
  memset(&a, 0, sizeof(a));
  a.grads = *grads; a.params = *params; a.sig = *sig; a.exp_avg = exp_avg; a.exp_avg_sq = exp_avg_sq; a.n_vec = n_vec;
  a.s = *s; a.scale = scale; a.rank = rank; a.world = world; a.zero_grad = zero_grad;
  const dim3 grid = shard_grid(n_vec, world, max_blocks);
  using namespace b2;
  if (bf16) sharded_step_kernel<true, ShardedAdamwUpdate><<<grid, kShardThreads, 0, stream>>>(a);
  else sharded_step_kernel<false, ShardedAdamwUpdate><<<grid, kShardThreads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

// The grouped steps: `map` holds this rank's group ids, one per fp32 parameter vector of its slice (n_vec / world x 1 (x 2)),
// and `gs` the scalars of n_groups groups.  Also cudaErrorInvalidValue, without a launch, for a null map or n_groups outside
// 1..64; the ids themselves are checked on the host where the map is built.
int b2_sharded_sgd_grouped_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const b2::SignalPads* sig,
                                  float* momentum, const uint8_t* map, const b2::SgdGroups* gs, int n_groups, size_t n_vec, float mu,
                                  int nesterov, float scale, int zero_grad, int rank, int world, int max_blocks,
                                  cudaStream_t stream) {
  if (momentum == nullptr || map == nullptr || gs == nullptr || n_groups < 1 || n_groups > b2::kMaxGroups ||
      !shard_args_ok(grads, params, sig, n_vec, rank, world))
    return (int)cudaErrorInvalidValue;
  b2::ShardedSgdGroupedArgs a;
  memset(&a, 0, sizeof(a));
  a.grads = *grads; a.params = *params; a.sig = *sig; a.momentum = momentum; a.map = map; a.n_vec = n_vec;
  a.mu = mu; a.scale = scale; a.rank = rank; a.world = world; a.zero_grad = zero_grad; a.gs = *gs;
  const dim3 grid = shard_grid(n_vec, world, max_blocks);
  using namespace b2;
  if (bf16) {
    if (nesterov) sharded_step_kernel<true, ShardedSgdGroupedUpdate<true>><<<grid, kShardThreads, 0, stream>>>(a);
    else sharded_step_kernel<true, ShardedSgdGroupedUpdate<false>><<<grid, kShardThreads, 0, stream>>>(a);
  } else {
    if (nesterov) sharded_step_kernel<false, ShardedSgdGroupedUpdate<true>><<<grid, kShardThreads, 0, stream>>>(a);
    else sharded_step_kernel<false, ShardedSgdGroupedUpdate<false>><<<grid, kShardThreads, 0, stream>>>(a);
  }
  return (int)cudaGetLastError();
}

int b2_sharded_adamw_grouped_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const b2::SignalPads* sig,
                                    float* exp_avg, float* exp_avg_sq, const uint8_t* map, const b2::AdamwScalars* s,
                                    const b2::AdamwGroups* gs, int n_groups, size_t n_vec, float scale, int zero_grad, int rank,
                                    int world, int max_blocks, cudaStream_t stream) {
  if (exp_avg == nullptr || exp_avg_sq == nullptr || map == nullptr || s == nullptr || gs == nullptr || n_groups < 1 ||
      n_groups > b2::kMaxGroups || !shard_args_ok(grads, params, sig, n_vec, rank, world))
    return (int)cudaErrorInvalidValue;
  b2::ShardedAdamwGroupedArgs a;
  memset(&a, 0, sizeof(a));
  a.grads = *grads; a.params = *params; a.sig = *sig; a.exp_avg = exp_avg; a.exp_avg_sq = exp_avg_sq; a.map = map;
  a.n_vec = n_vec; a.s = *s; a.gs = *gs; a.scale = scale; a.rank = rank; a.world = world; a.zero_grad = zero_grad;
  const dim3 grid = shard_grid(n_vec, world, max_blocks);
  using namespace b2;
  if (bf16) sharded_step_kernel<true, ShardedAdamwGroupedUpdate><<<grid, kShardThreads, 0, stream>>>(a);
  else sharded_step_kernel<false, ShardedAdamwGroupedUpdate><<<grid, kShardThreads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

// The capturable steps (Capturable<U>): as the launchers above, with the scalars taken from the block `blk` on the device.
// `map`: null without groups, else this rank's group ids.  Same grid, same refusals, and a null block is refused too.
int b2_sharded_sgd_cap_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const b2::SignalPads* sig, float* momentum,
                              const uint8_t* map, const b2::FlatScalars* blk, size_t n_vec, float mu, int nesterov, float scale,
                              int zero_grad, int rank, int world, int max_blocks, cudaStream_t stream) {
  if (momentum == nullptr || blk == nullptr || !shard_args_ok(grads, params, sig, n_vec, rank, world))
    return (int)cudaErrorInvalidValue;
  using namespace b2;
  const dim3 grid = shard_grid(n_vec, world, max_blocks);
  if (map != nullptr) {
    CapArgs<ShardedSgdGroupedArgs> a;
    memset(&a, 0, sizeof(a));
    a.grads = *grads; a.params = *params; a.sig = *sig; a.momentum = momentum; a.map = map; a.n_vec = n_vec;
    a.mu = mu; a.scale = scale; a.rank = rank; a.world = world; a.zero_grad = zero_grad; a.blk = blk;
    if (bf16) {
      if (nesterov) sharded_step_kernel<true, Capturable<ShardedSgdGroupedUpdate<true>>><<<grid, kShardThreads, 0, stream>>>(a);
      else sharded_step_kernel<true, Capturable<ShardedSgdGroupedUpdate<false>>><<<grid, kShardThreads, 0, stream>>>(a);
    } else {
      if (nesterov) sharded_step_kernel<false, Capturable<ShardedSgdGroupedUpdate<true>>><<<grid, kShardThreads, 0, stream>>>(a);
      else sharded_step_kernel<false, Capturable<ShardedSgdGroupedUpdate<false>>><<<grid, kShardThreads, 0, stream>>>(a);
    }
    return (int)cudaGetLastError();
  }
  CapArgs<ShardedSgdArgs> a;
  memset(&a, 0, sizeof(a));
  a.grads = *grads; a.params = *params; a.sig = *sig; a.momentum = momentum; a.n_vec = n_vec;
  a.mu = mu; a.scale = scale; a.rank = rank; a.world = world; a.zero_grad = zero_grad; a.blk = blk;
  if (bf16) {
    if (nesterov) sharded_step_kernel<true, Capturable<ShardedSgdUpdate<true>>><<<grid, kShardThreads, 0, stream>>>(a);
    else sharded_step_kernel<true, Capturable<ShardedSgdUpdate<false>>><<<grid, kShardThreads, 0, stream>>>(a);
  } else {
    if (nesterov) sharded_step_kernel<false, Capturable<ShardedSgdUpdate<true>>><<<grid, kShardThreads, 0, stream>>>(a);
    else sharded_step_kernel<false, Capturable<ShardedSgdUpdate<false>>><<<grid, kShardThreads, 0, stream>>>(a);
  }
  return (int)cudaGetLastError();
}

int b2_sharded_adamw_cap_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const b2::SignalPads* sig, float* exp_avg,
                                float* exp_avg_sq, const uint8_t* map, const b2::FlatScalars* blk, size_t n_vec, float scale,
                                int zero_grad, int rank, int world, int max_blocks, cudaStream_t stream) {
  if (exp_avg == nullptr || exp_avg_sq == nullptr || blk == nullptr || !shard_args_ok(grads, params, sig, n_vec, rank, world))
    return (int)cudaErrorInvalidValue;
  using namespace b2;
  const dim3 grid = shard_grid(n_vec, world, max_blocks);
  if (map != nullptr) {
    CapArgs<ShardedAdamwGroupedArgs> a;
    memset(&a, 0, sizeof(a));
    a.grads = *grads; a.params = *params; a.sig = *sig; a.exp_avg = exp_avg; a.exp_avg_sq = exp_avg_sq; a.map = map;
    a.n_vec = n_vec; a.scale = scale; a.rank = rank; a.world = world; a.zero_grad = zero_grad; a.blk = blk;
    if (bf16) sharded_step_kernel<true, Capturable<ShardedAdamwGroupedUpdate>><<<grid, kShardThreads, 0, stream>>>(a);
    else sharded_step_kernel<false, Capturable<ShardedAdamwGroupedUpdate>><<<grid, kShardThreads, 0, stream>>>(a);
    return (int)cudaGetLastError();
  }
  CapArgs<ShardedAdamwArgs> a;
  memset(&a, 0, sizeof(a));
  a.grads = *grads; a.params = *params; a.sig = *sig; a.exp_avg = exp_avg; a.exp_avg_sq = exp_avg_sq; a.n_vec = n_vec;
  a.scale = scale; a.rank = rank; a.world = world; a.zero_grad = zero_grad; a.blk = blk;
  if (bf16) sharded_step_kernel<true, Capturable<ShardedAdamwUpdate>><<<grid, kShardThreads, 0, stream>>>(a);
  else sharded_step_kernel<false, Capturable<ShardedAdamwUpdate>><<<grid, kShardThreads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

// The steps with RMSprop (FlatRMSprop): `square_avg` is this rank's shard (n_vec / world x 4 (x 8) floats), and `grad_avg` /
// `momentum_buffer` its shards of the centered average and the momentum buffer, or null when the update is not centered / has
// no momentum (s->centered / s->momentum are set here from them).  `map`: null without groups, else this rank's group ids with
// `gs` the lr and weight decay of n_groups groups.  Same grid, same refusals, and also cudaErrorInvalidValue, without a launch,
// for n_groups outside 1..64 with a map.
int b2_sharded_rmsprop_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const b2::SignalPads* sig, float* square_avg,
                              float* grad_avg, float* momentum_buffer, const uint8_t* map, const b2::RmspropScalars* s,
                              const b2::SgdGroups* gs, int n_groups, size_t n_vec, float scale, int zero_grad, int rank, int world,
                              int max_blocks, cudaStream_t stream) {
  if (square_avg == nullptr || s == nullptr || !shard_args_ok(grads, params, sig, n_vec, rank, world)) return (int)cudaErrorInvalidValue;
  using namespace b2;
  const dim3 grid = shard_grid(n_vec, world, max_blocks);
  if (map != nullptr) {
    if (gs == nullptr || n_groups < 1 || n_groups > kMaxGroups) return (int)cudaErrorInvalidValue;
    ShardedRmspropGroupedArgs a;
    memset(&a, 0, sizeof(a));
    a.grads = *grads; a.params = *params; a.sig = *sig; a.square_avg = square_avg; a.grad_avg = grad_avg;
    a.momentum_buffer = momentum_buffer; a.map = map; a.n_vec = n_vec; a.s = *s; a.gs = *gs; a.scale = scale; a.rank = rank;
    a.world = world; a.zero_grad = zero_grad;
    a.s.centered = grad_avg != nullptr ? 1 : 0;
    a.s.momentum = momentum_buffer != nullptr ? 1 : 0;
    if (bf16) sharded_step_kernel<true, ShardedRmspropGroupedUpdate><<<grid, kShardThreads, 0, stream>>>(a);
    else sharded_step_kernel<false, ShardedRmspropGroupedUpdate><<<grid, kShardThreads, 0, stream>>>(a);
    return (int)cudaGetLastError();
  }
  ShardedRmspropArgs a;
  memset(&a, 0, sizeof(a));
  a.grads = *grads; a.params = *params; a.sig = *sig; a.square_avg = square_avg; a.grad_avg = grad_avg;
  a.momentum_buffer = momentum_buffer; a.n_vec = n_vec; a.s = *s; a.scale = scale; a.rank = rank; a.world = world;
  a.zero_grad = zero_grad;
  a.s.centered = grad_avg != nullptr ? 1 : 0;
  a.s.momentum = momentum_buffer != nullptr ? 1 : 0;
  if (bf16) sharded_step_kernel<true, ShardedRmspropUpdate><<<grid, kShardThreads, 0, stream>>>(a);
  else sharded_step_kernel<false, ShardedRmspropUpdate><<<grid, kShardThreads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

// The capturable RMSprop steps (Capturable<U>): lr and weight decay (with `map`: every group's) from the block `blk`, alpha,
// 1 - alpha, eps and momentum from `s`.  Same refusals, and a null block is refused too.
int b2_sharded_rmsprop_cap_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const b2::SignalPads* sig,
                                  float* square_avg, float* grad_avg, float* momentum_buffer, const uint8_t* map,
                                  const b2::FlatScalars* blk, const b2::RmspropScalars* s, size_t n_vec, float scale, int zero_grad,
                                  int rank, int world, int max_blocks, cudaStream_t stream) {
  if (square_avg == nullptr || s == nullptr || blk == nullptr || !shard_args_ok(grads, params, sig, n_vec, rank, world))
    return (int)cudaErrorInvalidValue;
  using namespace b2;
  const dim3 grid = shard_grid(n_vec, world, max_blocks);
  if (map != nullptr) {
    CapArgs<ShardedRmspropGroupedArgs> a;
    memset(&a, 0, sizeof(a));
    a.grads = *grads; a.params = *params; a.sig = *sig; a.square_avg = square_avg; a.grad_avg = grad_avg;
    a.momentum_buffer = momentum_buffer; a.map = map; a.n_vec = n_vec; a.s = *s; a.scale = scale; a.rank = rank;
    a.world = world; a.zero_grad = zero_grad; a.blk = blk;
    a.s.centered = grad_avg != nullptr ? 1 : 0;
    a.s.momentum = momentum_buffer != nullptr ? 1 : 0;
    if (bf16) sharded_step_kernel<true, Capturable<ShardedRmspropGroupedUpdate>><<<grid, kShardThreads, 0, stream>>>(a);
    else sharded_step_kernel<false, Capturable<ShardedRmspropGroupedUpdate>><<<grid, kShardThreads, 0, stream>>>(a);
    return (int)cudaGetLastError();
  }
  CapArgs<ShardedRmspropArgs> a;
  memset(&a, 0, sizeof(a));
  a.grads = *grads; a.params = *params; a.sig = *sig; a.square_avg = square_avg; a.grad_avg = grad_avg;
  a.momentum_buffer = momentum_buffer; a.n_vec = n_vec; a.s = *s; a.scale = scale; a.rank = rank; a.world = world;
  a.zero_grad = zero_grad; a.blk = blk;
  a.s.centered = grad_avg != nullptr ? 1 : 0;
  a.s.momentum = momentum_buffer != nullptr ? 1 : 0;
  if (bf16) sharded_step_kernel<true, Capturable<ShardedRmspropUpdate>><<<grid, kShardThreads, 0, stream>>>(a);
  else sharded_step_kernel<false, Capturable<ShardedRmspropUpdate>><<<grid, kShardThreads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

}  // extern "C"
