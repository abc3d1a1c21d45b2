// Shared device helpers for the sm_90a kernels (inline PTX; no CUTLASS dependency).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <cstdio>

#define B2_MAX_RANKS 8
#define B2_MAX_BLOCKS 160            // signal-pad rows (>= largest comm grid)
#define B2_SIGNAL_WORDS (B2_MAX_BLOCKS * B2_MAX_RANKS + B2_MAX_BLOCKS + 64)

#ifndef B2_SPIN_LIMIT
#define B2_SPIN_LIMIT (1ull << 26)   // bounded spin (~tens of seconds), then trap with a diagnostic
#endif

struct PeerPtrs {                    // passed by value: per-rank base pointers of one symmetric buffer
  void* p[B2_MAX_RANKS];
};

namespace b2 {

// ----------------------------------------------------------------- programmatic dependent launch (PDL)
// launch_dependents: the next kernel in the stream/graph may start launching now (its CTAs then park in pdl_wait);
// pdl_wait: blocks until the previous kernel has completed and its writes are visible.  Both are no-ops when the
// kernel was launched without the programmatic-serialization attribute.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ----------------------------------------------------------------- memory model helpers
__device__ __forceinline__ void st_release_sys(uint32_t* addr, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* addr) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys(uint32_t* addr, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* addr) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }

// 16-byte global accesses that bypass L1 (peer data must never be served from a stale L1 line)
__device__ __forceinline__ uint4 ld_cg_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void st_cg_v4(void* p, uint4 v) {
  asm volatile("st.global.cg.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

// 16-byte volatile accesses for flag-in-data ("LL") exchanges: one store / one load instruction per line, never cached in
// L1, so a line that crossed NVLink is observed old or new per 8-byte half (the reader checks both flags)
__device__ __forceinline__ void st_volatile_v4(void* p, uint4 v) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ uint4 ld_volatile_v4(const void* p) {
  uint4 r;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}

// NVLS: in-switch reduction / broadcast on a multicast address (SASS: LDGMC / STGMC... )
__device__ __forceinline__ float4 multimem_ld_reduce_f32x4(const void* mc) {
  float4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(mc) : "memory");
  return r;
}
__device__ __forceinline__ uint4 multimem_ld_reduce_bf16x8(const void* mc) {
  uint4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(mc) : "memory");
  return r;
}
__device__ __forceinline__ void multimem_st_v4(void* mc, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(__uint_as_float(v.x)),
               "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w)) : "memory");
}

// ----------------------------------------------------------------- bf16 <-> fp32 packing
__device__ __forceinline__ float bf16lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// ----------------------------------------------------------------- Philox4x32-10 (counter based RNG)
struct Philox {
  __device__ static __forceinline__ uint4 gen(uint64_t seed, uint64_t subseq, uint64_t offset) {
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    uint4 c = make_uint4((uint32_t)offset, (uint32_t)(offset >> 32), (uint32_t)subseq, (uint32_t)(subseq >> 32));
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
      uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
      c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    return c;
  }
};

// ----------------------------------------------------------------- cross-GPU block barrier
// Signal pad (uint32 words) of every rank:  flags[B2_MAX_BLOCKS][B2_MAX_RANKS] | epoch[B2_MAX_BLOCKS]
// Block b of rank r signals block b of every peer by writing the new epoch into the peer's
// flags[b][r]; it then waits until its own flags[b][q] reached that epoch for every q.  Epochs only
// grow (wrap-safe signed compare), so one slot per (block, source) suffices: a peer can be at most one
// barrier ahead of us.  Release/acquire at .sys scope orders the data accesses around the barrier.
struct SignalPads {
  uint32_t* pad[B2_MAX_RANKS];
};

__device__ __forceinline__ uint32_t barrier_epoch_load(const SignalPads& s, int rank) {
  return s.pad[rank][B2_MAX_BLOCKS * B2_MAX_RANKS + blockIdx.x];
}
__device__ __forceinline__ void barrier_epoch_store(const SignalPads& s, int rank, uint32_t e) {
  s.pad[rank][B2_MAX_BLOCKS * B2_MAX_RANKS + blockIdx.x] = e;
}

// All threads of the block must call this. `epoch` is the value to publish (previous + 1).
__device__ __forceinline__ void block_barrier_all_ranks(const SignalPads& s, int rank, int world, uint32_t epoch) {
  __syncthreads();
  if (threadIdx.x < (unsigned)world) {
    const int peer = threadIdx.x;
    st_release_sys(s.pad[peer] + blockIdx.x * B2_MAX_RANKS + rank, epoch);
    const uint32_t* mine = s.pad[rank] + blockIdx.x * B2_MAX_RANKS + peer;
    unsigned long long spins = 0;
    // (acquire loads in the loop rather than relaxed polling + one fence.acq_rel.sys afterwards: the sys-scope fence
    //  is the more expensive of the two)
    while ((int32_t)(ld_acquire_sys(mine) - epoch) < 0) {
      if (++spins > B2_SPIN_LIMIT) {
        printf("[b200dist] barrier timeout: rank %d block %d waiting for rank %d epoch %u (have %u)\n", rank,
               (int)blockIdx.x, peer, epoch, ld_relaxed_sys(mine));
        __trap();
      }
    }
  }
  __syncthreads();
}

}  // namespace b2
