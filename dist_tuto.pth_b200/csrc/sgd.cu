// Fused  [peer-memory gradient all-reduce] + [1/world scale] + [momentum SGD]  for flat fp32 buffers.
//
// Replaces average_gradients() + optimizer.step() + optimizer.zero_grad() of the reference training
// step (train_dist.py:118,123,124): 8 all-reduces + 8 divides + foreach-SGD + 8 memsets become ONE
// kernel, in two exchange flavours with identical arithmetic (fixed rank order => bit-identical replicas):
//   * allreduce_sgd_push_kernel (default for world > 1): every rank stores its locally reduced bucket, flag-in-data,
//     into every peer's inbox over NVSwitch and reduces out of its own memory -- one NVLink crossing on the critical path;
//   * allreduce_sgd_kernel: flag barrier, then every rank loads all peers' buckets (one-shot).  Also the world == 1 path.
// Both apply  buf = mu*buf + g ; p -= lr*buf  (torch.optim.SGD semantics with dampening 0 -- train_dist.py:110), or, in their
// SgdArgsGeneral instances, the same with torch's weight decay and Nesterov momentum (sgd_device.cuh), re-zero the gradient bucket of the other step parity for the next `red.add` accumulation,
// keep conv2.weight pre-arranged for the step kernels (`aux`) and bump the device step counter used by the dropout RNG.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "common.cuh"
#include "sgd_device.cuh"
#include "convnet_reduce.cuh"
#include "param_groups.cuh"
#include "flat_scalars.cuh"

namespace b2 {

// Args: SgdArgs, SgdArgsGeneral (weight decay / Nesterov) or SgdArgsClip (+ gradient-norm clipping).  The clip instance asks
// for one CTA per SM (its grid is at most 64 CTAs): aimed at two, ptxas gives it 64 registers and it spills.
template <class Args>
__global__ void __launch_bounds__(kSgdThreads, kClipArgs<Args> ? 1 : 0) allreduce_sgd_kernel(Args a) {
  const int rank = a.rank, world = a.world;
  // Step parity (which gradient bucket is live) + step bump.  Thread 0 of every block reads the counter and then
  // checks in with an atomic; the LAST block to check in knows every block has read it and bumps it right away, so
  // the atomic's latency hides behind the rest of the kernel and no block can see the new value.
  __shared__ unsigned int s_par;
  __shared__ float s_lr;
  pdl_wait();                        // gradients of this step (previous kernel) are complete and visible
  pdl_launch_dependents();           // the next step's forward/backward kernel may pre-launch now (it zeroes its smem, then waits)
  const unsigned long long t_waited = a.phase_ts != nullptr ? globaltimer() : 0ull;
  snapshot_loss(a);
  unsigned long long st = 0ull;
  unsigned int seen = 0u;
  if (threadIdx.x == 0) {
    st = a.step != nullptr ? *reinterpret_cast<volatile unsigned long long*>(a.step) : 0ull;
    s_par = (unsigned int)(st & 1ull);
    if (a.step != nullptr) seen = atomicAdd(a.done_counter, 1u);    // result is only consumed at the very end (latency hidden)
    s_lr = step_lr(a, st);
  }
  __syncthreads();
  const float lr = s_lr;
  uint32_t epoch = 0;
  if (world > 1) {
    epoch = barrier_epoch_load(a.sig, rank);
    block_barrier_all_ranks(a.sig, rank, world, ++epoch);           // all gradient buckets are complete
  }
  const size_t stride = (size_t)gridDim.x * kSgdThreads;
  // Double-buffered buckets remove the second barrier: once every rank has arrived at THIS step's barrier it has
  // finished reading last step's bucket, so that one can be zeroed right away for the step after this one.
  const bool dbuf = a.grad_stride > 0;
  const size_t par = dbuf ? (size_t)s_par : 0;
  const size_t cur_off = par * (size_t)a.grad_stride * sizeof(float);
  const size_t oth_off = (par ^ 1) * (size_t)a.grad_stride * sizeof(float);
  float sq = 0.f;                     // clip instance: this thread's sum of squares of the averaged gradient
  // block-uniform trip count (barrier inside the loop)
  for (size_t base = (size_t)blockIdx.x * kSgdThreads; base < a.n_vec; base += stride) {
    const size_t v = base + threadIdx.x;
    const bool ok = v < a.n_vec;
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ok) {
      uint4 raw[B2_MAX_RANKS];
#pragma unroll
      for (int r = 0; r < B2_MAX_RANKS; ++r)
        if (r < world) raw[r] = ld_cg_v4(reinterpret_cast<const uint4*>(reinterpret_cast<const char*>(a.grads.p[r]) + cur_off) + v);
#pragma unroll
      for (int r = 0; r < B2_MAX_RANKS; ++r)
        if (r < world) {
          g.x += __uint_as_float(raw[r].x); g.y += __uint_as_float(raw[r].y);
          g.z += __uint_as_float(raw[r].z); g.w += __uint_as_float(raw[r].w);
        }
      if constexpr (kClipArgs<Args>) clip_stash(a, v, g, sq);
      else sgd_apply(a, v, g, lr);
    }
    if (a.zero_grads) {
      if (dbuf) {
        if (ok) st_cg_v4(reinterpret_cast<uint4*>(reinterpret_cast<char*>(a.grads.p[rank]) + oth_off) + v, make_uint4(0u, 0u, 0u, 0u));
      } else {
        if (world > 1) block_barrier_all_ranks(a.sig, rank, world, ++epoch);   // peers are done reading this pass
        if (ok) st_cg_v4(reinterpret_cast<uint4*>(a.grads.p[rank]) + v, make_uint4(0u, 0u, 0u, 0u));
      }
    }
  }
  if (world > 1 && threadIdx.x == 0) barrier_epoch_store(a.sig, rank, epoch);
  if constexpr (kClipArgs<Args>) {   // phase B: every thread applies the vectors it stashed, clipped by the grid's norm
    const float coef = clip_grid_coef(a, sq);
    for (size_t v = (size_t)blockIdx.x * kSgdThreads + threadIdx.x; v < a.n_vec; v += stride) clip_apply(a, v, coef, lr);
  }
  if (a.phase_ts != nullptr) {
    __syncthreads();
    if (threadIdx.x == 0) {
      ts_put(a.phase_ts, st, (int)blockIdx.x, TS_OPT_WAITED, t_waited);
      ts_put(a.phase_ts, st, (int)blockIdx.x, TS_OPT_EXIT, globaltimer());
    }
  }
  // the last block to have checked in knows every block has read the step counter: it publishes step + 1
  if (threadIdx.x == 0 && a.step != nullptr && seen == gridDim.x - 1) { *a.done_counter = 0u; *a.step = st + 1ull; }
}

// World-1 optimizer of the per-sample step kernel run with per-CTA slots and fc1 factors (convnet.cu, convnet_args.cuh): every
// CTA reduces its share of the local gradient in a fixed order (convnet_reduce.cuh) and applies SGD to it straight from
// registers.  No bucket is read or red.add-ed, and the loss terms of the slots are summed in slot order, so the whole step is
// bit-reproducible.  Also bumps the step counter, snapshots the loss and refreshes aux like the kernels above, and re-zeroes the
// gradient bucket of the other step parity as they do (a.grads.p[0], optional): a trainer may still run a bucket step next (a
// batch on another path, such as the native executor's), and every bucket step relies on finding its bucket zeroed by the step
// before it.
//
// kSched: a.sched is a schedule (kind != LRS_NONE).  Thread 0 then also evaluates the step's lr where it waits for the
// step counter, and the emits read it from shared memory.  Without a schedule the kernel is compiled without that code:
// the fp64 schedule code costs this latency-bound kernel registers and instruction order even where it does not run.
// Args: SgdArgs, or SgdArgsGeneral for weight decay / Nesterov, compiled in for the same reason.  SgdArgsClip: phase A
// reduces every unit into the clip scratch (a CTA runs several units where the card has fewer than RED_UNITS SMs), and
// phase B applies the clipped gradient grid-stride after the grid barrier.
template <bool kSched, class Args>
__global__ void __launch_bounds__(cn::RED_T) reduce_sgd_kernel(Args a, const float* __restrict__ slots, int n_slots,
                                                               const float* __restrict__ factors, int n_samples, float* loss_acc) {
  __shared__ cn::RedSmem s;
  __shared__ unsigned long long s_step;
  __shared__ float s_lr;
  pdl_wait();                        // slots and factors of this step are complete and visible
  pdl_launch_dependents();
  const unsigned long long t_waited = a.phase_ts != nullptr ? globaltimer() : 0ull;
  // Thread 0 issues the step-counter read here.  It waits for the value, stores it and checks in on done_counter only once
  // its first unit's loads are in flight (RED_AT_ISSUED), so the read adds no round trip.  The check-in follows the read, so
  // no CTA can see the step + 1 that the last CTA to check in publishes.
  const unsigned long long st_read = threadIdx.x == 0 && a.step != nullptr ? *reinterpret_cast<volatile unsigned long long*>(a.step) : 0ull;
  unsigned int seen = 0u;
  if (blockIdx.x == 0 && threadIdx.x >= cn::RED_T - 32 && loss_acc != nullptr) {   // last warp of CTA 0 (no fc1 loads)
    const int i = threadIdx.x - (cn::RED_T - 32);
    const float prev = i < 2 ? loss_acc[i] : 0.f;    // in flight with the slot loads
    const float2 l = cn::reduce_loss(slots, n_slots);
    if (i < 2) {                     // the only writer of loss_acc while this kernel runs
      const float v = prev + (i == 0 ? l.x : l.y);
      loss_acc[i] = v;
      if (a.loss_snapshot != nullptr) a.loss_snapshot[i] = v;
    }
  }
  // momentum and parameters of the vectors a thread will update are loaded together with the unit's gradient terms
  // (clip instance: they are loaded in phase B)
  struct MP { float4 m, p; };
  struct NoMP {};
  unsigned long long t_mark[3] = {0ull, 0ull, 0ull};
  int last_unit = 0;
  float sq = 0.f;                    // clip instance: this thread's sum of squares of the local gradient
  cn::reduce_local_grad(
      slots, n_slots, factors, n_samples, (int)blockIdx.x, (int)gridDim.x, s,
      [&](int v) {
        if constexpr (kClipArgs<Args>) return NoMP{};
        else return MP{reinterpret_cast<const float4*>(a.momentum)[v], reinterpret_cast<const float4*>(a.params)[v]};
      },
      [&](int v, float4 g, const auto& h) {
        if constexpr (kClipArgs<Args>) clip_stash(a, (size_t)v, g, sq);
        else sgd_apply_mp(a, (size_t)v, g, h.m, h.p, kSched ? s_lr : a.lr);   // s_lr, s_step: written before the first barrier
        if (a.grads.p[0] != nullptr) {
          const size_t z = a.grad_stride > 0 ? (size_t)((s_step & 1ull) ^ 1ull) * (size_t)a.grad_stride : 0;
          st_cg_v4(reinterpret_cast<float*>(a.grads.p[0]) + z + (size_t)v * 4, make_uint4(0u, 0u, 0u, 0u));
        }
      },
      [&](int point, int u) {                            // thread 0 only
        if (point == cn::RED_AT_ISSUED && u == (int)blockIdx.x) {   // the CTA's first unit
          s_step = st_read;
          if (a.step != nullptr) seen = atomicAdd(a.done_counter, 1u);   // consumed at the very end (latency hidden)
          if (kSched) s_lr = step_lr(a, st_read);
        }
        if (a.phase_ts != nullptr) { t_mark[point] = globaltimer(); last_unit = u; }
      });
  __syncthreads();                   // s_step is visible to every thread
  const unsigned long long st = s_step;
  if constexpr (kClipArgs<Args>) {   // phase B
    const float coef = clip_grid_coef(a, sq);
    const float lr = kSched ? s_lr : a.lr;
    for (size_t v = (size_t)blockIdx.x * cn::RED_T + threadIdx.x; v < a.n_vec; v += (size_t)gridDim.x * cn::RED_T)
      clip_apply(a, v, coef, lr);
  }
  if (a.phase_ts != nullptr) {
    if (threadIdx.x == 0) {
      ts_put(a.phase_ts, st, (int)blockIdx.x, TS_OPT_UNIT, last_unit < cn::RED_FC1_TILES ? 1ull : 2ull);
      ts_put(a.phase_ts, st, (int)blockIdx.x, TS_OPT_LOADED, t_mark[cn::RED_AT_LOADED]);
      ts_put(a.phase_ts, st, (int)blockIdx.x, TS_OPT_EMITTED, t_mark[cn::RED_AT_EMITTED]);
      ts_put(a.phase_ts, st, (int)blockIdx.x, TS_OPT_WAITED, t_waited);
      ts_put(a.phase_ts, st, (int)blockIdx.x, TS_OPT_EXIT, globaltimer());
    }
  }
  if (threadIdx.x == 0 && a.step != nullptr && seen == gridDim.x - 1) { *a.done_counter = 0u; *a.step = st + 1ull; }
}

// Push ("LL") variant of the same step: no flag barrier and no remote loads.
//
// Every rank STORES its locally reduced bucket into every peer's inbox as 16-byte lines {v0, epoch, v1, epoch}
// (the flag travels with the data, so one NVLink crossing both delivers and publishes it), then sums the world lines of
// each element out of its OWN memory, polling until both flags of a line carry this step's epoch.  Compared with
// barrier + peer loads (flag crossing, then a load round trip) the critical path is ONE one-way crossing.  The sum
// runs in fixed rank order with the own contribution taken from registers at position `rank`, so replicas stay
// bit-identical and equal to the barrier variant.  epoch = step + 1 (its wrap to 0, the value of a freshly zeroed line,
// is sent as 1: epoch 1 has the other parity); lines are double-buffered by step parity: a peer can only write parity p
// again two steps later, which needs my push of the step in between, which I issue after I finished reading parity p.
// The SgdArgsGeneral instance asks for one CTA per SM: left to itself ptxas aims that instance at three 512-thread CTAs per
// SM, 40 registers, and spills; the grid (<= 64 CTAs) never needs more than one per SM.  0: the default instance's bounds.
// The SgdArgsClip instance (the same bounds) stashes the vectors in phase A and applies them after the grid barrier.
template <class Args>
__global__ void __launch_bounds__(kSgdThreads, std::is_same<Args, SgdArgs>::value ? 0 : 1) allreduce_sgd_push_kernel(Args a) {
  __shared__ unsigned long long s_step;
  __shared__ float s_lr;
  pdl_wait();
  pdl_launch_dependents();
  snapshot_loss(a);
  unsigned int seen = 0u;
  if (threadIdx.x == 0) {
    s_step = *reinterpret_cast<volatile unsigned long long*>(a.step);
    seen = atomicAdd(a.done_counter, 1u);
    s_lr = step_lr(a, s_step);
  }
  __syncthreads();
  const unsigned long long st = s_step;
  const float lr = s_lr;
  const size_t stride = (size_t)gridDim.x * kSgdThreads;
  if constexpr (kClipArgs<Args>) {
    float sq = 0.f;
    for (size_t v = (size_t)blockIdx.x * kSgdThreads + threadIdx.x; v < a.n_vec; v += stride) exchange_apply_vec(a, v, st, lr, &sq);
    const float coef = clip_grid_coef(a, sq);
    for (size_t v = (size_t)blockIdx.x * kSgdThreads + threadIdx.x; v < a.n_vec; v += stride) clip_apply(a, v, coef, lr);
  } else {
    for (size_t v = (size_t)blockIdx.x * kSgdThreads + threadIdx.x; v < a.n_vec; v += stride) exchange_apply_vec(a, v, st, lr);
  }
  if (threadIdx.x == 0 && seen == gridDim.x - 1) { *a.done_counter = 0u; *a.step = st + 1ull; }
}

// Deterministic mode of the fused ConvNet step (convnet_args.cuh: det_partials): every step CTA stored its gradient sums to a
// private slot; this kernel adds the slots IN CTA ORDER into this step's bucket, so the local sum -- and with the fixed rank
// order of the exchange the whole update -- is bit-reproducible from run to run (float red.add into one bucket is not).
__global__ void __launch_bounds__(256) det_reduce_kernel(const float* __restrict__ partials, int n_slots, long long slot_stride,
                                                         float* __restrict__ grads, const unsigned long long* __restrict__ step,
                                                         long long grad_stride, int n_vec, float* __restrict__ loss_acc) {
  pdl_wait();
  pdl_launch_dependents();
  const int v = blockIdx.x * 256 + threadIdx.x;
  if (v == n_vec && loss_acc != nullptr) {        // the vector behind the parameters: {batch-mean nll, #correct} of every CTA
    float l = 0.f, c = 0.f;
    for (int sl = 0; sl < n_slots; ++sl) {
      l += __ldcg(partials + (size_t)sl * slot_stride + (size_t)n_vec * 4);
      c += __ldcg(partials + (size_t)sl * slot_stride + (size_t)n_vec * 4 + 1);
    }
    loss_acc[0] += l;                             // the only writer of loss_acc while this kernel runs
    loss_acc[1] += c;
  }
  if (v >= n_vec) return;
  const unsigned long long st = step != nullptr ? *step : 0ull;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int sl = 0; sl < n_slots; ++sl) {
    const float4 q = __ldcg(reinterpret_cast<const float4*>(partials + (size_t)sl * slot_stride) + v);
    acc.x += q.x; acc.y += q.y; acc.z += q.z; acc.w += q.w;
  }
  reinterpret_cast<float4*>(grads + (size_t)(st & 1ull) * (size_t)grad_stride)[v] = acc;
}

// Plain flat momentum SGD (generic models: gradients already averaged in `grad`).  kNesterov: step along g + mu*m instead of m.
// kScaled: the gradient is g * amp_inv_scale(grad_scale) (sgd_device.cuh); the kScaled = false instances never read grad_scale.
template <bool kNesterov, bool kScaled>
__global__ void __launch_bounds__(256) sgd_flat_kernel(float* __restrict__ p, float* __restrict__ m,
                                                       const float* __restrict__ g, size_t n, float lr, float mu,
                                                       float wd, int zero_grad, float* gw, const float* grad_scale) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n4 = n / 4;
  const float inv = kScaled ? amp_inv_scale(grad_scale) : 1.f;
  if (i < n4) {
    float4 gv = reinterpret_cast<const float4*>(g)[i];
    float4 pv = reinterpret_cast<float4*>(p)[i];
    float4 mv = reinterpret_cast<float4*>(m)[i];
    if constexpr (kScaled) gv = amp_unscale4(gv, inv);
    gv.x = fmaf(wd, pv.x, gv.x); gv.y = fmaf(wd, pv.y, gv.y); gv.z = fmaf(wd, pv.z, gv.z); gv.w = fmaf(wd, pv.w, gv.w);
    mv.x = fmaf(mu, mv.x, gv.x); mv.y = fmaf(mu, mv.y, gv.y); mv.z = fmaf(mu, mv.z, gv.z); mv.w = fmaf(mu, mv.w, gv.w);
    float4 dv = mv;
    if (kNesterov) {
      dv.x = fmaf(mu, mv.x, gv.x); dv.y = fmaf(mu, mv.y, gv.y); dv.z = fmaf(mu, mv.z, gv.z); dv.w = fmaf(mu, mv.w, gv.w);
    }
    pv.x = fmaf(-lr, dv.x, pv.x); pv.y = fmaf(-lr, dv.y, pv.y); pv.z = fmaf(-lr, dv.z, pv.z); pv.w = fmaf(-lr, dv.w, pv.w);
    reinterpret_cast<float4*>(p)[i] = pv;
    reinterpret_cast<float4*>(m)[i] = mv;
    if (zero_grad) reinterpret_cast<float4*>(gw)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (i == 0) {
    for (size_t t = n4 * 4; t < n; ++t) {      // tail (< 4 elements)
      const float gt = fmaf(wd, p[t], kScaled ? amp_unscale(g[t], inv) : g[t]);
      m[t] = fmaf(mu, m[t], gt);
      p[t] = fmaf(-lr, kNesterov ? fmaf(mu, m[t], gt) : m[t], p[t]);
      if (zero_grad) gw[t] = 0.f;
    }
  }
}

// FlatSGD's clipping, part 1: the sum of squares of one bucket's gradient g[0, n) into sqnorms[k] (fp64).  Each thread sums
// its squares in fp32 (its float4 vectors in order; thread 0 of CTA 0 also the < 4 tail elements), each CTA in a fixed
// tree, and the last CTA to finish adds the CTA partials in CTA order in fp64.  ws: [kClipMaxCtas partials | ticket], the
// ticket zero between calls (the last CTA resets it).  kScaled: the squares of g * amp_inv_scale(grad_scale).
constexpr int kSqnormThreads = 256;
template <bool kScaled>
__global__ void __launch_bounds__(kSqnormThreads) grad_sqnorm_kernel(const float* __restrict__ g, size_t n, float* ws,
                                                                      double* __restrict__ sqnorms, int k, const float* grad_scale) {
  __shared__ float s_part[kClipMaxCtas];
  __shared__ int s_last;
  const size_t n4 = n / 4;
  const float inv = kScaled ? amp_inv_scale(grad_scale) : 1.f;
  float sq = 0.f;
  for (size_t i = (size_t)blockIdx.x * kSqnormThreads + threadIdx.x; i < n4; i += (size_t)gridDim.x * kSqnormThreads) {
    float4 v = reinterpret_cast<const float4*>(g)[i];
    if constexpr (kScaled) v = amp_unscale4(v, inv);
    sq = fmaf(v.x, v.x, sq); sq = fmaf(v.y, v.y, sq); sq = fmaf(v.z, v.z, sq); sq = fmaf(v.w, v.w, sq);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0)
    for (size_t t = n4 * 4; t < n; ++t) {
      const float gt = kScaled ? amp_unscale(g[t], inv) : g[t];
      sq = fmaf(gt, gt, sq);
    }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, d);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = sq;
  __syncthreads();
  unsigned int* ticket = reinterpret_cast<unsigned int*>(ws + kClipMaxCtas);
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < kSqnormThreads / 32; ++w) t += s_part[w];
    __stcg(ws + blockIdx.x, t);
    __threadfence();
    s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    if (s_last) __threadfence();
  }
  __syncthreads();
  if (!s_last) return;
  if (threadIdx.x < gridDim.x) s_part[threadIdx.x] = __ldcg(ws + threadIdx.x);
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < (int)gridDim.x; ++i) s += (double)s_part[i];
    sqnorms[k] = s;
    *ticket = 0u;
  }
}

// FlatSGD's clipping, part 2: sgd_flat_kernel's update of one bucket after g *= coef, where coef comes from the total norm
// sqrt(sum of sqnorms[0, n_buckets) in bucket order), taken in fp64 and rounded once to fp32 (grad_norm_out, optional).
template <bool kNesterov, bool kScaled>
__global__ void __launch_bounds__(256) sgd_flat_clip_kernel(float* __restrict__ p, float* __restrict__ m,
                                                            const float* __restrict__ g, size_t n, float lr, float mu,
                                                            float wd, int zero_grad, float* gw, const double* __restrict__ sqnorms,
                                                            int n_buckets, float max_norm, float* grad_norm_out,
                                                            const float* grad_scale) {
  __shared__ float s_coef;
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int k = 0; k < n_buckets; ++k) s += sqnorms[k];
    const float nrm = __double2float_rn(__dsqrt_rn(s));
    s_coef = clip_coef(nrm, max_norm);
    if (blockIdx.x == 0 && grad_norm_out != nullptr) *grad_norm_out = nrm;
  }
  __syncthreads();
  const float c = s_coef;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n4 = n / 4;
  const float inv = kScaled ? amp_inv_scale(grad_scale) : 1.f;
  if (i < n4) {
    float4 gv = reinterpret_cast<const float4*>(g)[i];
    float4 pv = reinterpret_cast<float4*>(p)[i];
    float4 mv = reinterpret_cast<float4*>(m)[i];
    if constexpr (kScaled) gv = amp_unscale4(gv, inv);
    gv.x = __fmul_rn(gv.x, c); gv.y = __fmul_rn(gv.y, c); gv.z = __fmul_rn(gv.z, c); gv.w = __fmul_rn(gv.w, c);
    gv.x = fmaf(wd, pv.x, gv.x); gv.y = fmaf(wd, pv.y, gv.y); gv.z = fmaf(wd, pv.z, gv.z); gv.w = fmaf(wd, pv.w, gv.w);
    mv.x = fmaf(mu, mv.x, gv.x); mv.y = fmaf(mu, mv.y, gv.y); mv.z = fmaf(mu, mv.z, gv.z); mv.w = fmaf(mu, mv.w, gv.w);
    float4 dv = mv;
    if (kNesterov) {
      dv.x = fmaf(mu, mv.x, gv.x); dv.y = fmaf(mu, mv.y, gv.y); dv.z = fmaf(mu, mv.z, gv.z); dv.w = fmaf(mu, mv.w, gv.w);
    }
    pv.x = fmaf(-lr, dv.x, pv.x); pv.y = fmaf(-lr, dv.y, pv.y); pv.z = fmaf(-lr, dv.z, pv.z); pv.w = fmaf(-lr, dv.w, pv.w);
    reinterpret_cast<float4*>(p)[i] = pv;
    reinterpret_cast<float4*>(m)[i] = mv;
    if (zero_grad) reinterpret_cast<float4*>(gw)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (i == 0) {
    for (size_t t = n4 * 4; t < n; ++t) {      // tail (< 4 elements)
      const float gt = fmaf(wd, p[t], __fmul_rn(kScaled ? amp_unscale(g[t], inv) : g[t], c));
      m[t] = fmaf(mu, m[t], gt);
      p[t] = fmaf(-lr, kNesterov ? fmaf(mu, m[t], gt) : m[t], p[t]);
      if (zero_grad) gw[t] = 0.f;
    }
  }
}

// sgd_flat_kernel / sgd_flat_clip_kernel with parameter groups: parameter vector i takes the lr and weight decay of group
// map[i] (param_groups.cuh); the tail (< 4 elements) shares the map entry of its vector.  The per-element sequence is the
// ungrouped kernels' (sgd4), so running those on each tensor's segment with its group's scalars gives the same bits.
template <bool kNesterov, bool kClip, bool kScaled>
__global__ void __launch_bounds__(256) sgd_flat_grouped_kernel(float* __restrict__ p, float* __restrict__ m,
                                                               const float* __restrict__ g, size_t n,
                                                               const uint8_t* __restrict__ map, SgdGroups gs, float mu,
                                                               int zero_grad, float* gw, const double* __restrict__ sqnorms,
                                                               int n_buckets, float max_norm, float* grad_norm_out,
                                                               const float* grad_scale) {
  float c = 1.f;
  if constexpr (kClip) {
    __shared__ float s_coef;
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int k = 0; k < n_buckets; ++k) s += sqnorms[k];
      const float nrm = __double2float_rn(__dsqrt_rn(s));
      s_coef = clip_coef(nrm, max_norm);
      if (blockIdx.x == 0 && grad_norm_out != nullptr) *grad_norm_out = nrm;
    }
    __syncthreads();
    c = s_coef;
  }
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n4 = n / 4;
  const float inv = kScaled ? amp_inv_scale(grad_scale) : 1.f;
  if (i < n4) {
    const int gid = map[i];
    float4 gv = reinterpret_cast<const float4*>(g)[i];
    float4 pv = reinterpret_cast<float4*>(p)[i];
    float4 mv = reinterpret_cast<float4*>(m)[i];
    if constexpr (kScaled) gv = amp_unscale4(gv, inv);
    if constexpr (kClip) {
      gv.x = __fmul_rn(gv.x, c); gv.y = __fmul_rn(gv.y, c); gv.z = __fmul_rn(gv.z, c); gv.w = __fmul_rn(gv.w, c);
    }
    sgd4<kNesterov>(pv, mv, gv, gs.lr[gid], mu, gs.wd[gid]);
    reinterpret_cast<float4*>(p)[i] = pv;
    reinterpret_cast<float4*>(m)[i] = mv;
    if (zero_grad) reinterpret_cast<float4*>(gw)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (i == 0 && n4 * 4 < n) {
    const int gid = map[n4];
    const float lr = gs.lr[gid], wd = gs.wd[gid];
    for (size_t t = n4 * 4; t < n; ++t) {      // tail (< 4 elements)
      const float gt = fmaf(wd, p[t], kClip ? __fmul_rn(kScaled ? amp_unscale(g[t], inv) : g[t], c)
                                            : (kScaled ? amp_unscale(g[t], inv) : g[t]));
      m[t] = fmaf(mu, m[t], gt);
      p[t] = fmaf(-lr, kNesterov ? fmaf(mu, m[t], gt) : m[t], p[t]);
      if (zero_grad) gw[t] = 0.f;
    }
  }
}

// Capturable instances of sgd_flat_kernel, sgd_flat_clip_kernel and sgd_flat_grouped_kernel (flat_scalars.cuh): the lr and
// weight decay (kGrouped: every group's) come from the scalar block `blk`, loaded once per CTA through shared memory, instead
// of the kernel arguments.  The per-element sequence is sgd4, the fmaf sequence of those kernels, so the same scalars give
// the same bits.  kScaled: GradScaler's step -- with found_inf != 0 only the zeroing (amp_skip_zero), else the gradient is
// g * amp_inv_scale(grad_scale) (grad_scale null: already unscaled).
template <bool kNesterov, bool kClip, bool kGrouped, bool kScaled>
__global__ void __launch_bounds__(256) sgd_flat_cap_kernel(float* __restrict__ p, float* __restrict__ m,
                                                           const float* __restrict__ g, size_t n, const uint8_t* __restrict__ map,
                                                           const FlatScalars* __restrict__ blk, float mu, int zero_grad, float* gw,
                                                           const double* __restrict__ sqnorms, int n_buckets, float max_norm,
                                                           float* grad_norm_out, const float* grad_scale, const float* found_inf) {
  __shared__ float s_coef, s_lr, s_wd;
  __shared__ SgdGroups s_gs;
  if constexpr (kScaled) {
    if (__ldg(found_inf) != 0.f) {
      amp_skip_zero(gw, n, zero_grad);
      return;
    }
  }
  const float inv = kScaled && grad_scale != nullptr ? amp_inv_scale(grad_scale) : 1.f;
  if constexpr (kGrouped) flat_block_load(s_gs, blk->sgd);
  if (threadIdx.x == 0) {
    if constexpr (!kGrouped) { s_lr = blk->lr; s_wd = blk->wd; }
    if constexpr (kClip) s_coef = flat_clip_coef(sqnorms, n_buckets, max_norm, grad_norm_out);
  }
  __syncthreads();
  const float c = kClip ? s_coef : 1.f;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n4 = n / 4;
  if (i < n4) {
    const int gid = kGrouped ? map[i] : 0;
    float4 gv = reinterpret_cast<const float4*>(g)[i];
    float4 pv = reinterpret_cast<float4*>(p)[i];
    float4 mv = reinterpret_cast<float4*>(m)[i];
    if constexpr (kScaled) gv = amp_unscale4(gv, inv);
    if constexpr (kClip) {
      gv.x = __fmul_rn(gv.x, c); gv.y = __fmul_rn(gv.y, c); gv.z = __fmul_rn(gv.z, c); gv.w = __fmul_rn(gv.w, c);
    }
    sgd4<kNesterov>(pv, mv, gv, kGrouped ? s_gs.lr[gid] : s_lr, mu, kGrouped ? s_gs.wd[gid] : s_wd);
    reinterpret_cast<float4*>(p)[i] = pv;
    reinterpret_cast<float4*>(m)[i] = mv;
    if (zero_grad) reinterpret_cast<float4*>(gw)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (i == 0 && n4 * 4 < n) {
    const int gid = kGrouped ? map[n4] : 0;
    const float lr = kGrouped ? s_gs.lr[gid] : s_lr, wd = kGrouped ? s_gs.wd[gid] : s_wd;
    for (size_t t = n4 * 4; t < n; ++t) {      // tail (< 4 elements)
      const float gt = fmaf(wd, p[t], kClip ? __fmul_rn(kScaled ? amp_unscale(g[t], inv) : g[t], c)
                                            : (kScaled ? amp_unscale(g[t], inv) : g[t]));
      m[t] = fmaf(mu, m[t], gt);
      p[t] = fmaf(-lr, kNesterov ? fmaf(mu, m[t], gt) : m[t], p[t]);
      if (zero_grad) gw[t] = 0.f;
    }
  }
}

// out[i] = the lr the optimizer kernels apply when the step counter reads steps[i] (tests tie it to ops/optim.LRSchedule)
__global__ void __launch_bounds__(256) lr_schedule_eval_kernel(LrSchedule s, float base, const long long* __restrict__ steps,
                                                               float* __restrict__ out, long long n) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i < n) out[i] = lr_schedule_lr(s, base, (unsigned long long)steps[i]);
}

}  // namespace b2

extern "C" {

// A clip instance waits for every CTA of its grid at the grid barrier, so the whole grid must be resident at once: refuse a
// grid the device cannot hold (`resident`: that kernel's resident-CTA capacity, computed once).
static int clip_grid_fits(const void* kernel, int threads, unsigned blocks, int* resident) {
  if (*resident == 0) {
    int dev = 0, sms = 0, per = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, kernel, threads, 0);
    if (e != cudaSuccess) return (int)e;
    *resident = per * sms;
  }
  return blocks <= (unsigned)b2::kClipMaxCtas && (int)blocks <= *resident ? 0 : (int)cudaErrorCooperativeLaunchTooLarge;
}

static unsigned long long* g_phase_ts = nullptr;   // opt-in phase timestamps (sgd_device.cuh: TS_STEPS); read at launch
void b2_set_phase_ts(unsigned long long* p) { g_phase_ts = p; }
unsigned long long* b2_phase_ts() { return g_phase_ts; }

int b2_allreduce_sgd_launch(const PeerPtrs* grads, const b2::SignalPads* sig, float* params, float* momentum,
                            unsigned long long* step, size_t n_elems, float lr, float mu, float scale, int rank,
                            int world, int zero_grads, long long grad_stride, unsigned int* done_counter, float* aux,
                            const PeerPtrs* inbox, const float* loss_acc, float* loss_snapshot, int wire_bf16,
                            const b2::LrSchedule* sched, float wd, int nesterov, float max_norm, float* clip_ws,
                            float* grad_norm_out, cudaStream_t stream) {
  if (world < 1 || world > B2_MAX_RANKS || rank < 0 || rank >= world) return (int)cudaErrorInvalidValue;
  if (!(wd >= 0.f)) return (int)cudaErrorInvalidValue;
  const bool clip = max_norm > 0.f;     // max_norm 0: no clipping
  if (clip && (clip_ws == nullptr || !(max_norm < INFINITY))) return (int)cudaErrorInvalidValue;
  b2::SgdArgsClip a;
  a.wd = wd; a.nesterov = nesterov ? 1 : 0;
  a.max_norm = max_norm; a.clip_ws = clip_ws; a.grad_norm_out = grad_norm_out;
  a.phase_ts = g_phase_ts;
  memset(&a.sched, 0, sizeof(a.sched));
  if (sched != nullptr) a.sched = *sched;
  a.wire_bf16 = wire_bf16;
  a.loss_acc = loss_acc; a.loss_snapshot = (loss_acc != nullptr) ? loss_snapshot : nullptr;
  memset(&a.inbox, 0, sizeof(a.inbox));
  // push ("LL") exchange: needs an inbox on every rank, the double-buffered buckets and the device step counter (its epoch)
  const bool push = inbox != nullptr && world > 1;
  if (push) {
    if (step == nullptr || grad_stride <= 0) return (int)cudaErrorInvalidValue;
    a.inbox = *inbox;
  }
  a.grads = *grads; a.sig = *sig; a.params = params; a.momentum = momentum; a.step = step;
  a.n_vec = n_elems / 4; a.lr = lr; a.mu = mu; a.scale = scale; a.rank = rank; a.world = world;
  a.zero_grads = zero_grads; a.grad_stride = grad_stride; a.done_counter = done_counter; a.aux = aux;
  if (step != nullptr && done_counter == nullptr) return (int)cudaErrorInvalidValue;
  size_t blocks = (a.n_vec + b2::kSgdThreads - 1) / b2::kSgdThreads;
  if (blocks < 1) blocks = 1;
  if (blocks > 64) blocks = 64;
  static const int pdl = [] { const char* e = getenv("B200DIST_PDL"); return (e == nullptr || e[0] != '0') ? 1 : 0; }();
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)blocks);
  cfg.blockDim = dim3((unsigned)b2::kSgdThreads);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  const b2::SgdArgs& plain = a;    // the default instances take SgdArgs alone
  const b2::SgdArgsGeneral& general = a;
  if (!clip) {
    if (wd != 0.f || nesterov)
      return push ? (int)cudaLaunchKernelEx(&cfg, b2::allreduce_sgd_push_kernel<b2::SgdArgsGeneral>, general)
                  : (int)cudaLaunchKernelEx(&cfg, b2::allreduce_sgd_kernel<b2::SgdArgsGeneral>, general);
    return push ? (int)cudaLaunchKernelEx(&cfg, b2::allreduce_sgd_push_kernel<b2::SgdArgs>, plain)
                : (int)cudaLaunchKernelEx(&cfg, b2::allreduce_sgd_kernel<b2::SgdArgs>, plain);
  }
  static int resident_push = 0, resident_pull = 0;
  const int rc = push ? clip_grid_fits((const void*)b2::allreduce_sgd_push_kernel<b2::SgdArgsClip>, b2::kSgdThreads,
                                       (unsigned)blocks, &resident_push)
                      : clip_grid_fits((const void*)b2::allreduce_sgd_kernel<b2::SgdArgsClip>, b2::kSgdThreads,
                                       (unsigned)blocks, &resident_pull);
  if (rc != 0) return rc;
  return push ? (int)cudaLaunchKernelEx(&cfg, b2::allreduce_sgd_push_kernel<b2::SgdArgsClip>, a)
              : (int)cudaLaunchKernelEx(&cfg, b2::allreduce_sgd_kernel<b2::SgdArgsClip>, a);
}

int b2_reduce_sgd_launch(float* params, float* momentum, unsigned long long* step, unsigned int* done_counter, float lr, float mu,
                         float* aux, float* loss_acc, float* loss_snapshot, const float* slots, int n_slots, const float* factors,
                         int n_samples, float* grads, long long grad_stride, const b2::LrSchedule* sched, float wd, int nesterov,
                         float max_norm, float* clip_ws, float* grad_norm_out, int n_cta, cudaStream_t stream) {
  if (step != nullptr && done_counter == nullptr) return (int)cudaErrorInvalidValue;
  if (n_cta < 0 || n_cta > cn::RED_UNITS) return (int)cudaErrorInvalidValue;
  if (!(wd >= 0.f)) return (int)cudaErrorInvalidValue;
  const bool clip = max_norm > 0.f;     // max_norm 0: no clipping
  if (clip && (clip_ws == nullptr || !(max_norm < INFINITY))) return (int)cudaErrorInvalidValue;
  b2::SgdArgsClip a;
  memset(&a, 0, sizeof(a));
  a.wd = wd; a.nesterov = nesterov ? 1 : 0;
  a.max_norm = max_norm; a.clip_ws = clip_ws; a.grad_norm_out = grad_norm_out;
  if (sched != nullptr) a.sched = *sched;
  a.params = params; a.momentum = momentum; a.step = step; a.done_counter = done_counter; a.aux = aux;
  a.n_vec = cn::NPAR / 4; a.lr = lr; a.mu = mu; a.scale = 1.f; a.rank = 0; a.world = 1;
  a.loss_acc = loss_acc; a.loss_snapshot = loss_acc != nullptr ? loss_snapshot : nullptr;
  a.grads.p[0] = grads; a.grad_stride = grad_stride;
  a.phase_ts = g_phase_ts;
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  // at most one CTA per SM; n_cta > 0 asks for that grid instead (a CTA then runs every n_cta-th unit, as on a smaller card)
  const int blocks = n_cta > 0 ? n_cta : (sms < cn::RED_UNITS ? sms : cn::RED_UNITS);
  static const int pdl = [] { const char* e = getenv("B200DIST_PDL"); return (e == nullptr || e[0] != '0') ? 1 : 0; }();
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)blocks);
  cfg.blockDim = dim3((unsigned)cn::RED_T);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  const b2::SgdArgs& plain = a;    // the default instances take SgdArgs alone
  const b2::SgdArgsGeneral& general = a;
  const bool sch = a.sched.kind != b2::LRS_NONE;
  if (!clip) {
    if (wd != 0.f || nesterov)
      return sch ? (int)cudaLaunchKernelEx(&cfg, b2::reduce_sgd_kernel<true, b2::SgdArgsGeneral>, general, slots, n_slots, factors,
                                           n_samples, loss_acc)
                 : (int)cudaLaunchKernelEx(&cfg, b2::reduce_sgd_kernel<false, b2::SgdArgsGeneral>, general, slots, n_slots, factors,
                                           n_samples, loss_acc);
    return sch ? (int)cudaLaunchKernelEx(&cfg, b2::reduce_sgd_kernel<true, b2::SgdArgs>, plain, slots, n_slots, factors, n_samples,
                                         loss_acc)
               : (int)cudaLaunchKernelEx(&cfg, b2::reduce_sgd_kernel<false, b2::SgdArgs>, plain, slots, n_slots, factors, n_samples,
                                         loss_acc);
  }
  static int resident = 0;         // one clip instance: a zero schedule gives the lr as it is
  const int rc = clip_grid_fits((const void*)b2::reduce_sgd_kernel<true, b2::SgdArgsClip>, cn::RED_T, (unsigned)blocks, &resident);
  if (rc != 0) return rc;
  return (int)cudaLaunchKernelEx(&cfg, b2::reduce_sgd_kernel<true, b2::SgdArgsClip>, a, slots, n_slots, factors, n_samples, loss_acc);
}

int b2_reduce_units() { return cn::RED_UNITS; }

int b2_det_reduce_launch(const float* partials, int n_slots, long long slot_stride, float* grads, const unsigned long long* step,
                         long long grad_stride, size_t n_elems, float* loss_acc, cudaStream_t stream) {
  const int n_vec = (int)(n_elems / 4);
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)((n_vec + 1 + 255) / 256));
  cfg.blockDim = dim3(256);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return (int)cudaLaunchKernelEx(&cfg, b2::det_reduce_kernel, partials, n_slots, slot_stride, grads, step, grad_stride, n_vec, loss_acc);
}

int b2_lr_schedule_eval_launch(const b2::LrSchedule* sched, float base, const long long* steps, float* out, long long n,
                               cudaStream_t stream) {
  if (n <= 0) return 0;
  b2::lr_schedule_eval_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(*sched, base, steps, out, n);
  return (int)cudaGetLastError();
}

// grad_scale (fp32 on the device, or null): GradScaler's loss scale, the scaled instances unscale the gradient as they load it.
int b2_sgd_flat_launch(float* p, float* m, const float* g, size_t n, float lr, float mu, float wd, int zero_grad, int nesterov,
                       float max_norm, const double* sqnorms, int n_buckets, float* grad_norm_out, const float* grad_scale,
                       cudaStream_t stream) {
  const size_t n4 = (n / 4) > 0 ? n / 4 : 1;
  const unsigned blocks = (unsigned)((n4 + 255) / 256);
  float* gw = const_cast<float*>(g);
  using namespace b2;
  const int k = (nesterov ? 2 : 0) | (grad_scale != nullptr ? 1 : 0);
  if (max_norm > 0.f) {            // clipped by the norm of grad_sqnorm's n_buckets sums (0: no clipping)
    if (sqnorms == nullptr || n_buckets < 1 || !(max_norm < INFINITY)) return (int)cudaErrorInvalidValue;
#define B2_SGD_CLIP(N, S) sgd_flat_clip_kernel<N, S><<<blocks, 256, 0, stream>>>(p, m, g, n, lr, mu, wd, zero_grad, gw, sqnorms, \
                                                                               n_buckets, max_norm, grad_norm_out, grad_scale)
    switch (k) {
      case 0: B2_SGD_CLIP(false, false); break;
      case 1: B2_SGD_CLIP(false, true); break;
      case 2: B2_SGD_CLIP(true, false); break;
      default: B2_SGD_CLIP(true, true); break;
    }
#undef B2_SGD_CLIP
    return (int)cudaGetLastError();
  }
#define B2_SGD(N, S) sgd_flat_kernel<N, S><<<blocks, 256, 0, stream>>>(p, m, g, n, lr, mu, wd, zero_grad, gw, grad_scale)
  switch (k) {
    case 0: B2_SGD(false, false); break;
    case 1: B2_SGD(false, true); break;
    case 2: B2_SGD(true, false); break;
    default: B2_SGD(true, true); break;
  }
#undef B2_SGD
  return (int)cudaGetLastError();
}

// sgd_flat with parameter groups: `map` holds one group id per parameter vector (ceil(n / 4) ids) and `gs` the scalars of
// n_groups groups.  cudaErrorInvalidValue, without a launch, for a null pointer, n_groups outside 1..64 or clipping without
// sqnorms; the ids themselves are checked on the host where the map is built.
int b2_sgd_flat_grouped_launch(float* p, float* m, const float* g, size_t n, const uint8_t* map, const b2::SgdGroups* gs,
                               int n_groups, float mu, int zero_grad, int nesterov, float max_norm, const double* sqnorms,
                               int n_buckets, float* grad_norm_out, const float* grad_scale, cudaStream_t stream) {
  if (p == nullptr || m == nullptr || g == nullptr || map == nullptr || gs == nullptr || n_groups < 1 ||
      n_groups > b2::kMaxGroups)
    return (int)cudaErrorInvalidValue;
  const bool clip = max_norm > 0.f;
  if (clip && (sqnorms == nullptr || n_buckets < 1 || !(max_norm < INFINITY))) return (int)cudaErrorInvalidValue;
  const size_t n4 = (n / 4) > 0 ? n / 4 : 1;
  const unsigned blocks = (unsigned)((n4 + 255) / 256);
  float* gw = const_cast<float*>(g);
  using namespace b2;
#define B2_SGD_GR(N, C, S) sgd_flat_grouped_kernel<N, C, S><<<blocks, 256, 0, stream>>>(p, m, g, n, map, *gs, mu, zero_grad, gw, \
      C ? sqnorms : nullptr, C ? n_buckets : 0, C ? max_norm : 0.f, C ? grad_norm_out : nullptr, grad_scale)
  const int k = (nesterov ? 4 : 0) | (clip ? 2 : 0) | (grad_scale != nullptr ? 1 : 0);
  switch (k) {
    case 0: B2_SGD_GR(false, false, false); break;
    case 1: B2_SGD_GR(false, false, true); break;
    case 2: B2_SGD_GR(false, true, false); break;
    case 3: B2_SGD_GR(false, true, true); break;
    case 4: B2_SGD_GR(true, false, false); break;
    case 5: B2_SGD_GR(true, false, true); break;
    case 6: B2_SGD_GR(true, true, false); break;
    default: B2_SGD_GR(true, true, true); break;
  }
#undef B2_SGD_GR
  return (int)cudaGetLastError();
}

// The capturable sgd_flat / sgd_flat_grouped (flat_scalars.cuh): the scalars come from the block `blk` on the device.  `map`:
// null without groups, else one group id per parameter vector.  cudaErrorInvalidValue, without a launch, for a null pointer
// or clipping without sqnorms.
// found_inf (fp32 on the device, or null): GradScaler's step, with grad_scale as in b2_sgd_flat_launch (null: already
// unscaled); without found_inf grad_scale must be null.
int b2_sgd_flat_cap_launch(float* p, float* m, const float* g, size_t n, const uint8_t* map, const b2::FlatScalars* blk, float mu,
                           int zero_grad, int nesterov, float max_norm, const double* sqnorms, int n_buckets, float* grad_norm_out,
                           const float* grad_scale, const float* found_inf, cudaStream_t stream) {
  if (found_inf == nullptr && grad_scale != nullptr) return (int)cudaErrorInvalidValue;
  if (p == nullptr || m == nullptr || g == nullptr || blk == nullptr) return (int)cudaErrorInvalidValue;
  const bool clip = max_norm > 0.f;
  if (clip && (sqnorms == nullptr || n_buckets < 1 || !(max_norm < INFINITY))) return (int)cudaErrorInvalidValue;
  const size_t n4 = (n / 4) > 0 ? n / 4 : 1;
  const unsigned blocks = (unsigned)((n4 + 255) / 256);
  float* gw = const_cast<float*>(g);
  using namespace b2;
#define B2_SGD_CAP(N, C, G, S) sgd_flat_cap_kernel<N, C, G, S><<<blocks, 256, 0, stream>>>(p, m, g, n, map, blk, mu, zero_grad, \
                                                          gw, sqnorms, n_buckets, max_norm, grad_norm_out, grad_scale, found_inf)
  const int k = (found_inf != nullptr ? 8 : 0) | (nesterov ? 4 : 0) | (clip ? 2 : 0) | (map != nullptr ? 1 : 0);
  switch (k) {
    case 0: B2_SGD_CAP(false, false, false, false); break;
    case 1: B2_SGD_CAP(false, false, true, false); break;
    case 2: B2_SGD_CAP(false, true, false, false); break;
    case 3: B2_SGD_CAP(false, true, true, false); break;
    case 4: B2_SGD_CAP(true, false, false, false); break;
    case 5: B2_SGD_CAP(true, false, true, false); break;
    case 6: B2_SGD_CAP(true, true, false, false); break;
    case 7: B2_SGD_CAP(true, true, true, false); break;
    case 8: B2_SGD_CAP(false, false, false, true); break;
    case 9: B2_SGD_CAP(false, false, true, true); break;
    case 10: B2_SGD_CAP(false, true, false, true); break;
    case 11: B2_SGD_CAP(false, true, true, true); break;
    case 12: B2_SGD_CAP(true, false, false, true); break;
    case 13: B2_SGD_CAP(true, false, true, true); break;
    case 14: B2_SGD_CAP(true, true, false, true); break;
    default: B2_SGD_CAP(true, true, true, true); break;
  }
#undef B2_SGD_CAP
  return (int)cudaGetLastError();
}

// ws: b2_grad_sqnorm_ws_floats() floats, zero before the first call
int b2_grad_sqnorm_ws_floats() { return b2::kClipMaxCtas + 4; }
int b2_grad_sqnorm_launch(const float* g, size_t n, float* ws, double* sqnorms, int k, const float* grad_scale,
                          cudaStream_t stream) {
  size_t blocks = (n / 4 + b2::kSqnormThreads - 1) / b2::kSqnormThreads;
  if (blocks < 1) blocks = 1;
  if (blocks > (size_t)b2::kClipMaxCtas) blocks = b2::kClipMaxCtas;
  if (grad_scale != nullptr)
    b2::grad_sqnorm_kernel<true><<<(unsigned)blocks, b2::kSqnormThreads, 0, stream>>>(g, n, ws, sqnorms, k, grad_scale);
  else
    b2::grad_sqnorm_kernel<false><<<(unsigned)blocks, b2::kSqnormThreads, 0, stream>>>(g, n, ws, sqnorms, k, nullptr);
  return (int)cudaGetLastError();
}

size_t b2_clip_ws_floats(size_t n_elems) { return b2::clip_ws_floats(n_elems / 4); }

}  // extern "C"
