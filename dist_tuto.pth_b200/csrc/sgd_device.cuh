// Device-side pieces of the fused [gradient exchange + 1/world + momentum SGD + re-zero] step of the optimizer kernels
// (sgd.cu), and the phase timestamps the step kernels (convnet.cu) share with them.
#pragma once
#include "common.cuh"
#include "lr_schedule.h"

namespace b2 {

constexpr int kSgdThreads = 512;

// Opt-in phase timestamps of the step (bench/step_phases.py; off unless a buffer is set with b2_set_phase_ts): thread 0 of
// every CTA writes %globaltimer (ns) into row [step % TS_STEPS][cta] of TS_PER_CTA words.  The step kernel uses words
// 0..10 (TS_ENTRY..TS_EXIT), the optimizer kernels words 11..15: reduce_sgd_kernel writes the kind of its last reduction unit
// (TS_OPT_UNIT: 1 = fc1.weight tile, 2 = other vectors; not a time) and when that unit's loads landed and its emit was done.
constexpr int TS_STEPS = 64, TS_CTAS = 256, TS_PER_CTA = 16;
enum : int { TS_ENTRY = 0, TS_WAITED, TS_S0, TS_S1, TS_S2, TS_S4, TS_S6, TS_S8A, TS_S8B, TS_FLUSHED, TS_EXIT,
             TS_OPT_UNIT = 11, TS_OPT_WAITED, TS_OPT_EXIT, TS_OPT_LOADED, TS_OPT_EMITTED };
static_assert(TS_EXIT < TS_OPT_UNIT && TS_OPT_EMITTED < TS_PER_CTA, "the step kernel's marks must stay in front of the optimizer's");
__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void ts_put(unsigned long long* ts, unsigned long long step, int cta, int k, unsigned long long t) {
  if (ts != nullptr && cta < TS_CTAS) ts[((step % TS_STEPS) * TS_CTAS + (unsigned long long)cta) * TS_PER_CTA + k] = t;
}

struct SgdArgs {
  PeerPtrs grads;            // symmetric flat fp32 gradient buckets (grads.p[rank] is ours)
  SignalPads sig;
  float* params;
  float* momentum;
  unsigned long long* step;  // incremented once per call (may be null)
  unsigned int* done_counter; // block-completion counter (device scratch, zero between calls)
  size_t n_vec;              // float4 vectors
  float lr, mu, scale;
  int rank, world;
  int zero_grads;
  long long grad_stride;     // > 0: two buckets, this step's bucket = step & 1; the OTHER bucket is re-zeroed here
  float* aux;                // optional [w2f 5000 | w2b 8000]: conv2.weight re-arranged for the forward/backward kernels
  PeerPtrs inbox;            // push variant only: every rank's inbox  [2 parities][world sources][n_vec][2 lines of 16 B]
  int wire_bf16;             // push variant: gradients cross NVLink as bf16 (ONE 16-byte line {2 x bf16x2 + 2 flags} per float4 vector
                             // instead of two), fp32 accumulation and fp32 master weights; every rank -- the sender included --
                             // sums the same rounded values, so replicas stay bit-identical
  const float* loss_acc;     // optional: the step kernels' running [sum of batch-mean nll, #correct] ...
  float* loss_snapshot;      // ... copied here (2 floats) = the cumulative loss as of THIS step (per-step D2H source)
  unsigned long long* phase_ts;   // optional phase timestamps (see TS_STEPS); nullptr: off
  LrSchedule sched;          // lr of the update = lr_schedule_lr(sched, lr, step counter); kind LRS_NONE: lr as it is
};

// The lr of the update run at step counter `st`; the kernels evaluate it in thread 0 and share it through shared memory.
__device__ __forceinline__ float step_lr(const SgdArgs& a, unsigned long long st) { return lr_schedule_lr(a.sched, a.lr, st); }

// The previous kernel of the stream (this step's forward/backward) is complete and the next step's kernel cannot pass its
// own griddepcontrol.wait before this kernel ends, so loss_acc holds exactly the loss up to and including this step.
__device__ __forceinline__ void snapshot_loss(const SgdArgs& a) {
  if (a.loss_snapshot != nullptr && blockIdx.x == 0 && threadIdx.x < 2)
    a.loss_snapshot[threadIdx.x] = *reinterpret_cast<const volatile float*>(a.loss_acc + threadIdx.x);
}

// SGD update of one float4 vector (+ the pre-arranged conv2.weight copies), shared by both exchange variants; sgd_apply_mp
// takes the vector's momentum and parameters already loaded; `lr` is this step's (step_lr)
__device__ __forceinline__ void sgd_apply_mp(const SgdArgs& a, size_t v, float4 g, float4 m, float4 p, float lr) {
  g.x *= a.scale; g.y *= a.scale; g.z *= a.scale; g.w *= a.scale;
  m.x = fmaf(a.mu, m.x, g.x); m.y = fmaf(a.mu, m.y, g.y); m.z = fmaf(a.mu, m.z, g.z); m.w = fmaf(a.mu, m.w, g.w);
  p.x = fmaf(-lr, m.x, p.x); p.y = fmaf(-lr, m.y, p.y); p.z = fmaf(-lr, m.z, p.z); p.w = fmaf(-lr, m.w, p.w);
  reinterpret_cast<float4*>(a.momentum)[v] = m;
  reinterpret_cast<float4*>(a.params)[v] = p;
  if (a.aux != nullptr && v >= 264 / 4 && v < (264 + 5000) / 4) {      // conv2.weight (flat offset 264, 5000 elements)
    const float pw[4] = {p.x, p.y, p.z, p.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int i = (int)v * 4 + e - 264;
      const int co = i / 250, r = i - co * 250, ci = r / 25, kk = r - ci * 25;
      a.aux[(ci * 25 + kk) * 20 + co] = pw[e];                                     // w2f [ci][ky][kx][co]
      a.aux[5000 + ((co * 25 + kk) * 2 + ci / 5) * 8 + ci % 5] = pw[e];            // w2b [co][ky][kx][half][8]
    }
  }
}
__device__ __forceinline__ void sgd_apply(const SgdArgs& a, size_t v, float4 g, float lr) {
  sgd_apply_mp(a, v, g, reinterpret_cast<const float4*>(a.momentum)[v], reinterpret_cast<const float4*>(a.params)[v], lr);
}

// One float4 vector `v` of the flat bucket through the push ("LL") exchange and the optimizer:
//   store my value, flag-in-data, into every peer's inbox (16-byte lines {v0, epoch, v1, epoch}); sum the world lines of this
//   vector out of MY inbox in fixed rank order (own contribution from registers) => bit-identical replicas; SGD; re-zero the
//   other-parity bucket.  world == 1: no exchange.  `st` = step index (flag = (uint32)(st + 1), or 1 where that wraps to 0;
//   parity = st & 1), `lr` = step_lr(a, st).
__device__ __forceinline__ void exchange_apply_vec(const SgdArgs& a, size_t v, unsigned long long st, float lr) {
  const int rank = a.rank, world = a.world;
  const uint32_t epoch = (uint32_t)(st + 1ull);
  const uint32_t flag = epoch == 0u ? 1u : epoch;                       // 0 is "never written"; epoch 1 has the other parity
  const size_t ipar = (size_t)(st & 1ull);                              // inbox lines are double-buffered by step parity
  const size_t par = a.grad_stride > 0 ? ipar : 0;                       // ... and so are the gradient buckets when there are two
  const size_t cur_off = par * (size_t)a.grad_stride * sizeof(float);
  const uint4 mine = ld_cg_v4(reinterpret_cast<const uint4*>(reinterpret_cast<const char*>(a.grads.p[rank]) + cur_off) + v);
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
  if (world > 1 && a.wire_bf16) {
    // one line per vector: {bf16(x),bf16(y) | flag | bf16(z),bf16(w) | flag}
    const uint32_t lo = pack_bf16x2(__uint_as_float(mine.x), __uint_as_float(mine.y));
    const uint32_t hi = pack_bf16x2(__uint_as_float(mine.z), __uint_as_float(mine.w));
    const uint4 l0 = make_uint4(lo, flag, hi, flag);
    const size_t dst_line = (ipar * (size_t)world + (size_t)rank) * a.n_vec + v;
#pragma unroll
    for (int i = 1; i < B2_MAX_RANKS; ++i) {
      if (i < world) {
        int r = rank + i;
        if (r >= world) r -= world;
        st_volatile_v4(reinterpret_cast<uint4*>(a.inbox.p[r]) + dst_line, l0);
      }
    }
    const uint4* in = reinterpret_cast<const uint4*>(a.inbox.p[rank]);
#pragma unroll
    for (int r = 0; r < B2_MAX_RANKS; ++r) {
      if (r < world) {
        uint4 q0;
        if (r == rank) {
          q0 = l0;
        } else {
          const uint4* src = in + (ipar * (size_t)world + (size_t)r) * a.n_vec + v;
          unsigned long long spins = 0;
          for (;;) {
            q0 = ld_volatile_v4(src);
            if (q0.y == flag && q0.w == flag) break;
            if (++spins > B2_SPIN_LIMIT) {
              printf("[b200dist] push all-reduce (bf16 wire): rank %d timed out waiting for rank %d (step %llu, vector %llu)\n", rank, r,
                     st, (unsigned long long)v);
              __trap();
            }
          }
        }
        g.x += bf16lo(q0.x); g.y += bf16hi(q0.x); g.z += bf16lo(q0.z); g.w += bf16hi(q0.z);
      }
    }
  } else if (world > 1) {
    const size_t dst_line = ((ipar * (size_t)world + (size_t)rank) * a.n_vec + v) * 2;   // ((parity * world + source) * n_vec + v) * 2
    const uint4 l0 = make_uint4(mine.x, flag, mine.y, flag), l1 = make_uint4(mine.z, flag, mine.w, flag);
#pragma unroll
    for (int i = 1; i < B2_MAX_RANKS; ++i) {          // start with the next rank so the ranks do not all hit one peer first
      if (i < world) {
        int r = rank + i;
        if (r >= world) r -= world;
        uint4* dst = reinterpret_cast<uint4*>(a.inbox.p[r]) + dst_line;
        st_volatile_v4(dst, l0);
        st_volatile_v4(dst + 1, l1);
      }
    }
    const uint4* in = reinterpret_cast<const uint4*>(a.inbox.p[rank]);
#pragma unroll
    for (int r = 0; r < B2_MAX_RANKS; ++r) {
      if (r < world) {
        uint4 q0, q1;
        if (r == rank) {
          q0 = l0; q1 = l1;
        } else {
          const uint4* src = in + ((ipar * (size_t)world + (size_t)r) * a.n_vec + v) * 2;
          unsigned long long spins = 0;
          for (;;) {
            q0 = ld_volatile_v4(src);
            q1 = ld_volatile_v4(src + 1);
            if (q0.y == flag && q0.w == flag && q1.y == flag && q1.w == flag) break;
            if (++spins > B2_SPIN_LIMIT) {
              printf("[b200dist] push all-reduce: rank %d timed out waiting for rank %d (step %llu, vector %llu)\n", rank, r, st,
                     (unsigned long long)v);
              __trap();
            }
          }
        }
        g.x += __uint_as_float(q0.x); g.y += __uint_as_float(q0.z);
        g.z += __uint_as_float(q1.x); g.w += __uint_as_float(q1.z);
      }
    }
  } else {
    g = make_float4(__uint_as_float(mine.x), __uint_as_float(mine.y), __uint_as_float(mine.z), __uint_as_float(mine.w));
  }
  sgd_apply(a, v, g, lr);
  if (a.zero_grads) {
    const size_t z_off = a.grad_stride > 0 ? (par ^ 1) * (size_t)a.grad_stride * sizeof(float) : 0;
    st_cg_v4(reinterpret_cast<uint4*>(reinterpret_cast<char*>(a.grads.p[rank]) + z_off) + v, make_uint4(0u, 0u, 0u, 0u));
  }
}

}  // namespace b2
