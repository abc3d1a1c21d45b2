// Fused  [peer-memory gradient all-reduce] + [1/world scale] + [momentum SGD]  for flat fp32 buffers.
//
// Replaces average_gradients() + optimizer.step() + optimizer.zero_grad() of the reference training
// step (train_dist.py:118,123,124): 8 all-reduces + 8 divides + foreach-SGD + 8 memsets become ONE
// kernel, in two exchange flavours with identical arithmetic (fixed rank order => bit-identical replicas):
//   * allreduce_sgd_push_kernel (default for world > 1): every rank stores its locally reduced bucket, flag-in-data,
//     into every peer's inbox over NVSwitch and reduces out of its own memory -- one NVLink crossing on the critical path;
//   * allreduce_sgd_kernel: flag barrier, then every rank loads all peers' buckets (one-shot).  Also the world == 1 path.
// Both apply  buf = mu*buf + g ; p -= lr*buf  (torch.optim.SGD semantics with dampening 0, no nesterov, no weight
// decay -- train_dist.py:110), re-zero the gradient bucket of the other step parity for the next `red.add` accumulation,
// keep conv2.weight pre-arranged for the step kernels (`aux`) and bump the device step counter used by the dropout RNG.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "common.cuh"
#include "sgd_device.cuh"
#include "convnet_reduce.cuh"

namespace b2 {

__global__ void __launch_bounds__(kSgdThreads) allreduce_sgd_kernel(SgdArgs a) {
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
      sgd_apply(a, v, g, lr);
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
template <bool kSched>
__global__ void __launch_bounds__(cn::RED_T) reduce_sgd_kernel(SgdArgs a, const float* __restrict__ slots, int n_slots,
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
  struct MP { float4 m, p; };
  unsigned long long t_mark[3] = {0ull, 0ull, 0ull};
  int last_unit = 0;
  cn::reduce_local_grad(
      slots, n_slots, factors, n_samples, (int)blockIdx.x, (int)gridDim.x, s,
      [&](int v) { return MP{reinterpret_cast<const float4*>(a.momentum)[v], reinterpret_cast<const float4*>(a.params)[v]}; },
      [&](int v, float4 g, const MP& h) {
        sgd_apply_mp(a, (size_t)v, g, h.m, h.p, kSched ? s_lr : a.lr);   // s_lr, s_step: written before the first barrier
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
__global__ void __launch_bounds__(kSgdThreads) allreduce_sgd_push_kernel(SgdArgs a) {
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
  for (size_t v = (size_t)blockIdx.x * kSgdThreads + threadIdx.x; v < a.n_vec; v += stride) exchange_apply_vec(a, v, st, lr);
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

// Plain flat momentum SGD (generic models: gradients already averaged in `grad`)
__global__ void __launch_bounds__(256) sgd_flat_kernel(float* __restrict__ p, float* __restrict__ m,
                                                       const float* __restrict__ g, size_t n, float lr, float mu,
                                                       float wd, int zero_grad, float* gw) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t n4 = n / 4;
  if (i < n4) {
    float4 gv = reinterpret_cast<const float4*>(g)[i];
    float4 pv = reinterpret_cast<float4*>(p)[i];
    float4 mv = reinterpret_cast<float4*>(m)[i];
    gv.x = fmaf(wd, pv.x, gv.x); gv.y = fmaf(wd, pv.y, gv.y); gv.z = fmaf(wd, pv.z, gv.z); gv.w = fmaf(wd, pv.w, gv.w);
    mv.x = fmaf(mu, mv.x, gv.x); mv.y = fmaf(mu, mv.y, gv.y); mv.z = fmaf(mu, mv.z, gv.z); mv.w = fmaf(mu, mv.w, gv.w);
    pv.x = fmaf(-lr, mv.x, pv.x); pv.y = fmaf(-lr, mv.y, pv.y); pv.z = fmaf(-lr, mv.z, pv.z); pv.w = fmaf(-lr, mv.w, pv.w);
    reinterpret_cast<float4*>(p)[i] = pv;
    reinterpret_cast<float4*>(m)[i] = mv;
    if (zero_grad) reinterpret_cast<float4*>(gw)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (i == 0) {
    for (size_t t = n4 * 4; t < n; ++t) {      // tail (< 4 elements)
      const float gt = fmaf(wd, p[t], g[t]);
      m[t] = fmaf(mu, m[t], gt);
      p[t] = fmaf(-lr, m[t], p[t]);
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

static unsigned long long* g_phase_ts = nullptr;   // opt-in phase timestamps (sgd_device.cuh: TS_STEPS); read at launch
void b2_set_phase_ts(unsigned long long* p) { g_phase_ts = p; }
unsigned long long* b2_phase_ts() { return g_phase_ts; }

int b2_allreduce_sgd_launch(const PeerPtrs* grads, const b2::SignalPads* sig, float* params, float* momentum,
                            unsigned long long* step, size_t n_elems, float lr, float mu, float scale, int rank,
                            int world, int zero_grads, long long grad_stride, unsigned int* done_counter, float* aux,
                            const PeerPtrs* inbox, const float* loss_acc, float* loss_snapshot, int wire_bf16,
                            const b2::LrSchedule* sched, cudaStream_t stream) {
  if (world < 1 || world > B2_MAX_RANKS || rank < 0 || rank >= world) return (int)cudaErrorInvalidValue;
  b2::SgdArgs a;
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
  return push ? (int)cudaLaunchKernelEx(&cfg, b2::allreduce_sgd_push_kernel, a)
              : (int)cudaLaunchKernelEx(&cfg, b2::allreduce_sgd_kernel, a);
}

int b2_reduce_sgd_launch(float* params, float* momentum, unsigned long long* step, unsigned int* done_counter, float lr, float mu,
                         float* aux, float* loss_acc, float* loss_snapshot, const float* slots, int n_slots, const float* factors,
                         int n_samples, float* grads, long long grad_stride, const b2::LrSchedule* sched, cudaStream_t stream) {
  if (step != nullptr && done_counter == nullptr) return (int)cudaErrorInvalidValue;
  b2::SgdArgs a;
  memset(&a, 0, sizeof(a));
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
  const int blocks = sms < cn::RED_UNITS ? sms : cn::RED_UNITS;   // at most one CTA per SM
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
  return a.sched.kind != b2::LRS_NONE
             ? (int)cudaLaunchKernelEx(&cfg, b2::reduce_sgd_kernel<true>, a, slots, n_slots, factors, n_samples, loss_acc)
             : (int)cudaLaunchKernelEx(&cfg, b2::reduce_sgd_kernel<false>, a, slots, n_slots, factors, n_samples, loss_acc);
}

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

int b2_sgd_flat_launch(float* p, float* m, const float* g, size_t n, float lr, float mu, float wd, int zero_grad,
                       cudaStream_t stream) {
  const size_t n4 = (n / 4) > 0 ? n / 4 : 1;
  const unsigned blocks = (unsigned)((n4 + 255) / 256);
  b2::sgd_flat_kernel<<<blocks, 256, 0, stream>>>(p, m, g, n, lr, mu, wd, zero_grad, const_cast<float*>(g));
  return (int)cudaGetLastError();
}

}  // extern "C"
