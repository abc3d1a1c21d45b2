// Native step executor: the training hot loop without the Python interpreter.
//
// The reference's hot loop (train_dist.py:115-124) is Python: DataLoader iteration, five framework calls and an
// optimizer step per batch.  Here the loop that feeds the GPU is C++ and software-pipelined over three streams:
//
//   copy stream    : ONE cudaMemcpyAsync per step -- the pinned loader slot [x | y] -> device input block[p]   (p = step & 1)
//   compute stream : waits for that copy, then replays a 2-kernel CUDA graph (convnet_step + allreduce_sgd) reading block[p]
//   d2h stream     : copies the running loss to the slot's pinned word; its event retires the step
//
// so the H2D copy of step i+1 and the loss read-back of step i-1 overlap the kernels of step i.  At most `max_in_flight`
// steps are outstanding; a retired step hands its slot back to the prefetch thread (loader.cpp).  The GIL is released
// around run().
//
// Chunk pipeline (the default when the loader ring is deep enough: num_slots >= 3K): K consecutive steps are issued together,
//   copy stream    : K cudaMemcpyAsync H2D        (that step's pinned loader slot -> device block g*K + j), then ONE event
//   compute stream : ONE graph of the K steps' kernels (a pure kernel chain: programmatic dependent launch stays intact across
//                    the K steps -- an H2D -> kernel edge in front of every step would cost as much as a graph
//                    boundary); captured once at construction
//   d2h stream     : K cudaMemcpyAsync D2H        (the cumulative loss after each step, snapshotted on the device by that
//                    step's optimizer tail into loss_hist[g*K + j] -> the step's pinned loss word)
// ordered by three events per chunk.  Chunk c+1's copies run while chunk c computes (two device block groups g), chunk
// c-1's losses drain meanwhile, and a loader slot goes back to the prefetch threads as soon as its H2D copy has completed
// (not when the step retires), so staging never waits for the GPU.  Every step still has its own H2D copy from pinned
// memory and its own D2H read-back; the per-step path remains for the steps that do not fill a chunk.
#include "executor.h"

#include <cuda.h>

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>

extern "C" {
int b2_convnet_step_launch(const float* params, float* grads, const void* x, int x_u8, const long long* target,
                           float* loss_acc, float* out_logp, float* mask_out, const unsigned long long* step,
                           unsigned long long seed, long long sample_base, int B, int training, int backward,
                           float inv_bsz, float p_drop, int max_ctas, long long grad_stride, const float* aux,
                           const void* tail, float* det_partials, float* factors, const unsigned int* in_flag,
                           unsigned int in_gen, int input_ready, cudaStream_t stream);
struct PeerPtrsC { void* p[8]; };
struct SignalPadsC { uint32_t* pad[8]; };
int b2_allreduce_sgd_launch(const PeerPtrsC* grads, const SignalPadsC* sig, float* params, float* momentum,
                            unsigned long long* step, size_t n_elems, float lr, float mu, float scale, int rank,
                            int world, int zero_grads, long long grad_stride, unsigned int* done_counter, float* aux,
                            const PeerPtrsC* inbox, const float* loss_acc, float* loss_snapshot, int wire_bf16,
                            unsigned int* snap_flag, unsigned int snap_gen, cudaStream_t stream);
int b2_reduce_sgd_launch(float* params, float* momentum, unsigned long long* step, unsigned int* done_counter, float lr, float mu,
                         float* aux, float* loss_acc, float* loss_snapshot, unsigned int* snap_flag, unsigned int snap_gen,
                         const float* slots, int n_slots, const float* factors, int n_samples, float* grads, long long grad_stride,
                         cudaStream_t stream);
int b2_convnet_cluster_launch(const float* params, float* grads, const void* x, int x_u8, const long long* target,
                              float* loss_acc, float* out_logp, float* mask_out, const unsigned long long* step,
                              unsigned long long seed, long long sample_base, int B, int training, int backward,
                              float inv_bsz, float p_drop, int cluster, int max_clusters, long long grad_stride,
                              const float* aux, const void* tail, float* det_partials, const unsigned int* in_flag,
                              unsigned int in_gen, cudaStream_t stream);
int b2_convnet_npar();
struct FusedTailHostC {            // mirrors cn::FusedTailHost (csrc/convnet_args.cuh)
  void* grad_ptrs[8];
  void* inbox_ptrs[8];
  float* params;
  float* momentum;
  unsigned long long* step;
  float* aux;
  const float* loss_acc;
  float* loss_snapshot;
  unsigned int* ticket;
  float lr, mu, scale;
  int rank, world;
  int wire_bf16;
};
}

namespace b2 {

// Stream memory operations (driver API, resolved at run time like csrc/symm_mem.cpp does): the copy stream publishes "batch
// landed" words the step kernels poll, the D2H stream waits on the "loss snapshot written" word the optimizer kernel sets.
using WriteValue32Fn = CUresult (*)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
using WaitValue32Fn = CUresult (*)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
static void* drv_sym(const char* name) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return fn;
}
static WriteValue32Fn p_write32() { static auto f = reinterpret_cast<WriteValue32Fn>(drv_sym("cuStreamWriteValue32")); return f; }
static WaitValue32Fn p_wait32() { static auto f = reinterpret_cast<WaitValue32Fn>(drv_sym("cuStreamWaitValue32")); return f; }

static inline long long now_ns() {
  return std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

StepExecutor::StepExecutor(const StepConfig& cfg, NativeLoader* loader, int max_in_flight)
    : cfg_(cfg), loader_(loader), max_in_flight_(max_in_flight < 1 ? 1 : max_in_flight) {
  cudaStreamCreateWithFlags(&copy_, cudaStreamNonBlocking);
  cudaStreamCreateWithFlags(&compute_, cudaStreamNonBlocking);
  cudaStreamCreateWithFlags(&d2h_, cudaStreamNonBlocking);
  for (int p = 0; p < 2; ++p) {
    cudaEventCreateWithFlags(&copied_[p], cudaEventDisableTiming);
    cudaEventCreateWithFlags(&kernels_done_[p], cudaEventDisableTiming);
    cudaEventCreateWithFlags(&loss_read_[p], cudaEventDisableTiming);
  }
  {
    const char* e = getenv("B200DIST_EXEC_DIRECT");
    direct_ = (e == nullptr || e[0] != '0');
  }
  {
    // flag mode of the per-slot ring path: no cross-stream events at all (see run()); needs the stream memory operations.
    // Opt-in (B200DIST_EXEC_FLAGS=1): an alternative to the event path, not the default.
    const char* e = getenv("B200DIST_EXEC_FLAGS");
    flags_ = (e != nullptr && e[0] == '1') && direct_ && cfg_.ring_base > 0 && cfg_.flags != nullptr && !cfg_.fused_tail &&
             cfg_.loss_hist != nullptr && p_write32() != nullptr && p_wait32() != nullptr;
    if (flags_) {      // probe: some driver configurations refuse memory operations on a stream
      if (p_write32()((CUstream)copy_, (CUdeviceptr)(uintptr_t)cfg_.flags, 0u, CU_STREAM_WRITE_VALUE_DEFAULT) != CUDA_SUCCESS ||
          cudaStreamSynchronize(copy_) != cudaSuccess) {
        cudaGetLastError();
        flags_ = false;
      }
    }
  }
  const int K = cfg_.chunk, nb = loader_->num_slots();
  chunk_ok_ = K >= 2 && K <= 8 && nb >= 3 * K && cfg_.loss_hist != nullptr;
  if (chunk_ok_) {
    for (int g = 0; g < 2; ++g) {
      cudaEventCreateWithFlags(&h2d_done_[g], cudaEventDisableTiming);
      cudaEventCreateWithFlags(&comp_done_[g], cudaEventDisableTiming);
      cudaEventCreateWithFlags(&d2h_done_[g], cudaEventDisableTiming);
    }
    copy_ev_.resize(nb + 2);
    for (auto& e : copy_ev_) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    for (int k = K; k >= 1 && n_sizes_ < 4; k /= 2) chunk_sizes_[n_sizes_++] = k;
  }
  slots_.resize(loader_->num_slots());
  for (auto& s : slots_) {
    cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming);
    cudaHostAlloc((void**)&s.loss_pin, 2 * sizeof(float), cudaHostAllocDefault);
    s.loss_pin[0] = s.loss_pin[1] = 0.f;
  }
}

StepExecutor::~StepExecutor() {
  drain();
  cudaStreamSynchronize(compute_);
  for (auto& s : slots_) {
    if (s.done) cudaEventDestroy(s.done);
    if (s.loss_pin) cudaFreeHost(s.loss_pin);
  }
  for (auto e : copy_ev_) if (e) cudaEventDestroy(e);
  for (int g = 0; g < 2; ++g) {
    for (int i = 0; i < 4; ++i) if (comp_exec_[g][i]) cudaGraphExecDestroy(comp_exec_[g][i]);
    if (h2d_done_[g]) cudaEventDestroy(h2d_done_[g]);
    if (comp_done_[g]) cudaEventDestroy(comp_done_[g]);
    if (d2h_done_[g]) cudaEventDestroy(d2h_done_[g]);
  }
  for (int p = 0; p < 2; ++p) {
    if (exec_[p]) cudaGraphExecDestroy(exec_[p]);
    if (copied_[p]) cudaEventDestroy(copied_[p]);
    if (kernels_done_[p]) cudaEventDestroy(kernels_done_[p]);
    if (loss_read_[p]) cudaEventDestroy(loss_read_[p]);
  }
  if (copy_) cudaStreamDestroy(copy_);
  if (compute_) cudaStreamDestroy(compute_);
  if (d2h_) cudaStreamDestroy(d2h_);
}

// Enqueues the two kernels of one step on the compute stream (called under stream capture).
void StepExecutor::record_step(const void* x, const long long* y, float* loss_snapshot, const unsigned int* in_flag,
                               unsigned int* snap_flag, unsigned int gen) {
  FusedTailHostC th;
  const void* tp = nullptr;
  if (cfg_.fused_tail) {
    std::memset(&th, 0, sizeof(th));
    std::memcpy(th.grad_ptrs, cfg_.grad_ptrs, sizeof(th.grad_ptrs));
    std::memcpy(th.inbox_ptrs, cfg_.inbox_ptrs, sizeof(th.inbox_ptrs));
    th.params = cfg_.params; th.momentum = cfg_.momentum; th.step = cfg_.step_counter; th.aux = cfg_.aux;
    th.loss_acc = cfg_.loss_acc; th.loss_snapshot = loss_snapshot; th.ticket = cfg_.ticket;
    th.lr = cfg_.lr; th.mu = cfg_.mu; th.scale = 1.f / cfg_.world; th.rank = cfg_.rank; th.world = cfg_.world;
    th.wire_bf16 = cfg_.wire_bf16;
    tp = &th;
  }
  // one GPU, one CTA per sample: plain stores to the slots / factors, reduced in a fixed order by the optimizer kernel
  const bool slots = cfg_.grad_slots != nullptr && cfg_.world == 1 && cfg_.cluster <= 1 && !cfg_.fused_tail;
  int rc = cfg_.cluster > 1
               ? b2_convnet_cluster_launch(cfg_.params, cfg_.grads_local, x, cfg_.x_u8, y, cfg_.loss_acc, nullptr, nullptr,
                                           cfg_.step_counter, cfg_.seed, cfg_.sample_base, cfg_.B, cfg_.training, 1,
                                           1.f / cfg_.B, cfg_.p_drop, cfg_.cluster, 0, cfg_.grad_stride, cfg_.aux, tp, nullptr, in_flag, gen, compute_)
               : b2_convnet_step_launch(cfg_.params, cfg_.grads_local, x, cfg_.x_u8, y, cfg_.loss_acc, nullptr, nullptr,
                                        cfg_.step_counter, cfg_.seed, cfg_.sample_base, cfg_.B, cfg_.training, 1, 1.f / cfg_.B,
                                        cfg_.p_drop, 0, cfg_.grad_stride, cfg_.aux, tp, slots ? cfg_.grad_slots : nullptr,
                                        slots ? cfg_.factors : nullptr, in_flag, gen, /*input_ready=*/1, compute_);
  int rc2 = 0;
  if (slots) {
    rc2 = b2_reduce_sgd_launch(cfg_.params, cfg_.momentum, cfg_.step_counter, cfg_.done_counter, cfg_.lr, cfg_.mu, cfg_.aux,
                               cfg_.loss_acc, loss_snapshot, snap_flag, gen, cfg_.grad_slots, cfg_.B, cfg_.factors, cfg_.B, cfg_.grads_local,
                               cfg_.grad_stride, compute_);
  } else if (!cfg_.fused_tail) {
    PeerPtrsC g;
    SignalPadsC sg;
    std::memcpy(g.p, cfg_.grad_ptrs, sizeof(g.p));
    std::memcpy(sg.pad, cfg_.sig_ptrs, sizeof(sg.pad));
    PeerPtrsC ib;
    std::memcpy(ib.p, cfg_.inbox_ptrs, sizeof(ib.p));
    rc2 = b2_allreduce_sgd_launch(&g, &sg, cfg_.params, cfg_.momentum, cfg_.step_counter, (size_t)b2_convnet_npar(),
                                  cfg_.lr, cfg_.mu, 1.f / cfg_.world, cfg_.rank, cfg_.world, 1, cfg_.grad_stride,
                                  cfg_.done_counter, cfg_.aux, cfg_.push ? &ib : nullptr, cfg_.loss_acc, loss_snapshot, cfg_.wire_bf16,
                                  snap_flag, gen, compute_);
  }
  if ((rc != 0 || rc2 != 0) && err_.empty())
    err_ = std::string("kernel launch failed: ") + cudaGetErrorString((cudaError_t)(rc ? rc : rc2));
}

bool StepExecutor::capture(int parity) {
  cudaGraph_t graph = nullptr;
  cudaError_t e = cudaStreamBeginCapture(compute_, cudaStreamCaptureModeThreadLocal);
  if (e != cudaSuccess) { err_ = std::string("cudaStreamBeginCapture: ") + cudaGetErrorString(e); return false; }
  err_.clear();
  record_step(cfg_.in_dev[parity], reinterpret_cast<const long long*>(cfg_.in_dev[parity] + loader_->y_offset()),
              cfg_.loss_hist != nullptr ? cfg_.loss_hist + 2 * parity : nullptr);
  e = cudaStreamEndCapture(compute_, &graph);
  if (!err_.empty() || e != cudaSuccess || graph == nullptr) {
    if (err_.empty()) err_ = std::string("graph capture failed: ") + cudaGetErrorString(e);
    if (graph) cudaGraphDestroy(graph);
    return false;
  }
  e = cudaGraphInstantiate(&exec_[parity], graph, 0);
  cudaGraphDestroy(graph);
  if (e != cudaSuccess) { err_ = std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e); return false; }
  return true;
}

// The three graphs of one chunk: loader slot group `sg` (pinned slots sg*K .. sg*K+K-1), device block group `g` (0/1).
static bool end_capture(cudaStream_t st, cudaGraphExec_t* out, std::string* err, const char* what) {
  cudaGraph_t graph = nullptr;
  cudaError_t e = cudaStreamEndCapture(st, &graph);
  if (!err->empty() || e != cudaSuccess || graph == nullptr) {
    if (err->empty()) *err = std::string(what) + " capture failed: " + cudaGetErrorString(e);
    if (graph) cudaGraphDestroy(graph);
    cudaGetLastError();
    return false;
  }
  e = cudaGraphInstantiate(out, graph, 0);
  cudaGraphDestroy(graph);
  if (e != cudaSuccess) { *err = std::string("cudaGraphInstantiate(") + what + "): " + cudaGetErrorString(e); cudaGetLastError(); return false; }
  return true;
}

bool StepExecutor::capture_chunk(int g, int si) {
  const int K = cfg_.chunk, k = chunk_sizes_[si];
  err_.clear();
  if (comp_exec_[g][si] != nullptr) return true;       // k steps' kernels: a pure chain, PDL intact from step to step
  cudaError_t e = cudaStreamBeginCapture(compute_, cudaStreamCaptureModeThreadLocal);
  if (e != cudaSuccess) { err_ = std::string("cudaStreamBeginCapture: ") + cudaGetErrorString(e); return false; }
  for (int j = 0; j < k; ++j) {
    unsigned char* blk = cfg_.in_dev[g * K + j];
    record_step(blk, reinterpret_cast<const long long*>(blk + loader_->y_offset()), cfg_.loss_hist + 2 * (g * K + j));
  }
  return end_capture(compute_, &comp_exec_[g][si], &err_, "compute chunk");
}

// Captures (and instantiates) every graph the hot loop replays, so that no capture lands inside a timed / training region.
bool StepExecutor::prepare() {
  if (!direct_)
    for (int p = 0; p < 2; ++p)
      if (exec_[p] == nullptr && !capture(p)) return false;
  if (chunk_ok_ && !direct_)
    for (int g = 0; g < 2 && chunk_ok_; ++g)
      for (int si = 0; si < n_sizes_; ++si)
        if (!capture_chunk(g, si)) { chunk_ok_ = false; chunk_note_ = err_; err_.clear(); break; }
  return true;
}

// Hand loader slots whose H2D copy has completed back to the prefetch threads (in hand-out order).
void StepExecutor::release_copied(bool block_for_one) {
  while (!copy_q_.empty()) {
    const CopyFlight& c = copy_q_.front();
    if (block_for_one) {
      const long long t0 = now_ns();
      cudaEventSynchronize(copy_ev_[c.ev]);
      stats_.copy_wait_ns += now_ns() - t0;
      block_for_one = false;
    }
    else if (cudaEventQuery(copy_ev_[c.ev]) != cudaSuccess) { cudaGetLastError(); break; }
    for (int j = 0; j < c.count; ++j) loader_->release();
    held_ -= c.count;
    copy_q_.pop_front();
  }
}

void StepExecutor::retire_oldest() {
  const Flight f = in_flight_.front();
  in_flight_.pop_front();
  const long long t0 = now_ns();
  cudaEventSynchronize(slots_[f.ev_slot].done);
  stats_.retire_ns += now_ns() - t0;
  const int s = f.slot;
  last_loss_ = (double)slots_[s].loss_pin[0];      // host read of this step's D2H loss copy
  if (!f.released_at_copy) loader_->release();
}

void StepExecutor::drain_copies() {
  while (!copy_q_.empty()) release_copied(true);
}

void StepExecutor::drain() {
  drain_copies();
  while (!in_flight_.empty()) retire_oldest();
  // flag mode retires a step when its loss snapshot has been read back, which the optimizer kernel allows as soon as it
  // has started: wait for the kernels themselves before the caller touches parameters or another stream takes over
  if (flags_) cudaStreamSynchronize(compute_);
}

int64_t StepExecutor::run(int64_t max_steps, int* pending_slot, int64_t* pending_count, int* epoch_done) {
  *pending_slot = -1;
  *pending_count = 0;
  *epoch_done = 0;
  int64_t done = 0;
  const int K = cfg_.chunk, nb = loader_->num_slots();
  struct Total { long long t0; Stats* s; ~Total() { s->total_ns += now_ns() - t0; } } total{now_ns(), &stats_};
  while (max_steps < 0 || done < max_steps) {
    // ---- chunk path: the largest chunk size (K, K/2, ...) that the budget and the epoch's full batches allow
    const int64_t room = std::min<int64_t>(max_steps < 0 ? K : max_steps - done, loader_->full_batches_left());
    int si = -1;
    for (int i = 0; i < n_sizes_; ++i)
      if (chunk_sizes_[i] <= room) { si = i; break; }
    if (chunk_ok_ && si >= 0) {
      const int kc = chunk_sizes_[si];
      const int g = (int)(chunks_issued_ & 1);
      if (!direct_ && comp_exec_[g][si] == nullptr && !capture_chunk(g, si)) {
        chunk_ok_ = false;
        chunk_note_ = err_;
        err_.clear();
        continue;
      }
      release_copied(false);
      while (held_ > nb - K) release_copied(true);                  // the prefetch threads need K free slots to stage into
      while ((int)in_flight_.size() > nb - K) retire_oldest();      // a slot's pinned loss word is reused nb steps later
      // copies: device block group g is free once the chunk that last read it (two chunks ago) has computed; blocks 0/1
      // are also the per-step path's double buffer
      cudaStreamWaitEvent(copy_, comp_done_[g], 0);
      cudaStreamWaitEvent(copy_, kernels_done_[0], 0);
      cudaStreamWaitEvent(copy_, kernels_done_[1], 0);
      int slot_of[8];
      for (int j = 0; j < kc; ++j) {                                // blocks until batch j is staged
        int64_t count = 0;
        const long long tn = now_ns();
        const int slot = loader_->next(&count);
        stats_.next_ns += now_ns() - tn;
        if (slot < 0 || count != cfg_.B) { err_ = "chunk path: loader handed out a short batch"; return -1; }
        slot_of[j] = slot;
        cudaMemcpyAsync(cfg_.in_dev[g * K + j], loader_->slot(slot).x, loader_->block_bytes(), cudaMemcpyHostToDevice, copy_);
      }
      const int ev = (int)(chunks_issued_ % (int64_t)copy_ev_.size());
      cudaEventRecord(copy_ev_[ev], copy_);
      cudaEventRecord(h2d_done_[g], copy_);
      copy_q_.push_back({ev, kc});
      held_ += kc;
      // kernels: after the copies, and after the losses of the chunk that last used snapshot group g have been read back
      cudaStreamWaitEvent(compute_, h2d_done_[g], 0);
      cudaStreamWaitEvent(compute_, d2h_done_[g], 0);
      if (direct_) {
        // plain PDL stream launches: the chunk only amortises the cross-stream events (3 per kc steps instead of 3 per step);
        // on the device the steps chain exactly as in per-step direct mode, with no graph boundary at all
        err_.clear();
        for (int j = 0; j < kc; ++j) {
          unsigned char* blk = cfg_.in_dev[g * K + j];
          record_step(blk, reinterpret_cast<const long long*>(blk + loader_->y_offset()), cfg_.loss_hist + 2 * (g * K + j));
        }
        if (!err_.empty()) return -1;
      } else {
        cudaError_t e = cudaGraphLaunch(comp_exec_[g][si], compute_);
        if (e != cudaSuccess) { err_ = std::string("cudaGraphLaunch(compute chunk): ") + cudaGetErrorString(e); return -1; }
      }
      cudaEventRecord(comp_done_[g], compute_);
      if (g == 0) { cudaEventRecord(kernels_done_[0], compute_); cudaEventRecord(kernels_done_[1], compute_); }
      // losses
      cudaStreamWaitEvent(d2h_, comp_done_[g], 0);
      for (int j = 0; j < kc; ++j)
        cudaMemcpyAsync(slots_[slot_of[j]].loss_pin, cfg_.loss_hist + 2 * (g * K + j), 2 * sizeof(float), cudaMemcpyDeviceToHost, d2h_);
      cudaEventRecord(d2h_done_[g], d2h_);
      cudaEventRecord(slots_[slot_of[kc - 1]].done, d2h_);
      for (int j = 0; j < kc; ++j) in_flight_.push_back({slot_of[j], slot_of[kc - 1], true});
      ++chunks_issued_;
      issued_ += kc;
      done += kc;
      stats_.chunk_steps += kc;
      continue;
    }
    drain_copies();                                                 // per-step path below releases at retire: keep the order
    while ((int)in_flight_.size() >= max_in_flight_) retire_oldest();
    int64_t count = 0;
    const long long tn1 = now_ns();
    const int slot = loader_->next(&count);
    stats_.next_ns += now_ns() - tn1;
    if (slot < 0) { *epoch_done = 1; break; }
    if (count != cfg_.B) {            // short tail batch: give it back to the caller (eager path)
      drain();
      cudaStreamSynchronize(compute_);
      *pending_slot = slot;
      *pending_count = count;
      break;
    }
    const int p = (int)(issued_ & 1);
    if (direct_ && cfg_.ring_base > 0) {
      // Per-slot device blocks and loss snapshots: a slot's block is rewritten only after the step that used it has
      // RETIRED (its D2H event was synchronised before the slot was released to the loader), so no device-side
      // "buffer free" events are needed -- 9 driver calls per step instead of 12 (the feeding thread shares a 16-core
      // quota with up to 8 ranks: calls per step are what bounds the end-to-end rate at 8 GPUs).
      unsigned char* blk = cfg_.in_dev[cfg_.ring_base + slot];
      float* snap = cfg_.loss_hist + 2 * (cfg_.ring_base + slot);
      if (flags_) {
        // Flag mode (opt-in): NO cross-stream event.  copy stream: H2D, then a stream memory op writes this step's generation
        // into the slot's "landed" word -- the step kernel polls it (convnet_args.cuh wait_input); compute stream: nothing but
        // the kernels, so step k+1's kernel pre-launches behind step k's optimizer kernel exactly as inside one CUDA graph
        // (an event wait between them cost ~3 us of device time per step); D2H stream: waits (stream memory op) for the
        // "snapshot written" word the optimizer kernel sets, then reads the loss.  7 driver calls per step.
        const unsigned int gen = (unsigned int)(issued_ + 1);
        unsigned int* in_flag = cfg_.flags + 2 * slot;
        unsigned int* snap_flag = cfg_.flags + 2 * slot + 1;
        cudaMemcpyAsync(blk, loader_->slot(slot).x, loader_->block_bytes(), cudaMemcpyHostToDevice, copy_);
        CUresult r1 = p_write32()((CUstream)copy_, (CUdeviceptr)(uintptr_t)in_flag, gen, CU_STREAM_WRITE_VALUE_DEFAULT);
        err_.clear();
        record_step(blk, reinterpret_cast<const long long*>(blk + loader_->y_offset()), snap, in_flag, snap_flag, gen);
        CUresult r2 = p_wait32()((CUstream)d2h_, (CUdeviceptr)(uintptr_t)snap_flag, gen, CU_STREAM_WAIT_VALUE_GEQ);
        if (r1 != CUDA_SUCCESS || r2 != CUDA_SUCCESS) {
          // without the write the kernel just launched would spin forever: publish the generation from the host side
          if (r1 != CUDA_SUCCESS) { cudaStreamSynchronize(copy_); cudaMemcpy(in_flag, &gen, sizeof(gen), cudaMemcpyHostToDevice); }
          if (err_.empty()) err_ = "stream memory operation failed (cuStreamWriteValue32 / cuStreamWaitValue32)";
          cudaStreamSynchronize(compute_);
          return -1;
        }
        if (!err_.empty()) return -1;
        cudaMemcpyAsync(slots_[slot].loss_pin, snap, 2 * sizeof(float), cudaMemcpyDeviceToHost, d2h_);
        cudaEventRecord(slots_[slot].done, d2h_);
        in_flight_.push_back({slot, slot, false});
        ++issued_;
        ++done;
        ++stats_.single_steps;
        continue;
      }
      cudaMemcpyAsync(blk, loader_->slot(slot).x, loader_->block_bytes(), cudaMemcpyHostToDevice, copy_);
      cudaEventRecord(copied_[p], copy_);
      cudaStreamWaitEvent(compute_, copied_[p], 0);
      err_.clear();
      record_step(blk, reinterpret_cast<const long long*>(blk + loader_->y_offset()), snap);
      if (!err_.empty()) return -1;
      cudaEventRecord(kernels_done_[p], compute_);
      cudaStreamWaitEvent(d2h_, kernels_done_[p], 0);
      cudaMemcpyAsync(slots_[slot].loss_pin, snap, 2 * sizeof(float), cudaMemcpyDeviceToHost, d2h_);
      cudaEventRecord(slots_[slot].done, d2h_);
      in_flight_.push_back({slot, slot, false});
      ++issued_;
      ++done;
      ++stats_.single_steps;
      continue;
    }
    if (!direct_ && exec_[p] == nullptr && !capture(p)) return -1;
    // H2D: block[p] is free once the kernels that last read it (two steps ago, or a chunk of group 0) are done
    cudaStreamWaitEvent(copy_, kernels_done_[p], 0);
    cudaMemcpyAsync(cfg_.in_dev[p], loader_->slot(slot).x, loader_->block_bytes(), cudaMemcpyHostToDevice, copy_);
    cudaEventRecord(copied_[p], copy_);
    // kernels.  direct mode (default): plain stream launches with the programmatic-dependent-launch attribute -- the steps
    // chain on the device exactly as inside one long graph (a graph launch per step costs device time at every
    // boundary); graph mode: one 2-kernel graph per step.
    cudaStreamWaitEvent(compute_, copied_[p], 0);
    float* snap = cfg_.loss_hist != nullptr ? cfg_.loss_hist + 2 * p : nullptr;
    if (snap != nullptr) cudaStreamWaitEvent(compute_, loss_read_[p], 0);   // snapshot slot p was read back (two steps ago)
    if (direct_) {
      err_.clear();
      record_step(cfg_.in_dev[p], reinterpret_cast<const long long*>(cfg_.in_dev[p] + loader_->y_offset()), snap);
      if (!err_.empty()) return -1;
    } else {
      cudaError_t e = cudaGraphLaunch(exec_[p], compute_);
      if (e != cudaSuccess) { err_ = std::string("cudaGraphLaunch: ") + cudaGetErrorString(e); return -1; }
    }
    cudaEventRecord(kernels_done_[p], compute_);
    // loss read-back: the cumulative loss as of THIS step (snapshotted on the device by the step's optimizer kernel)
    cudaStreamWaitEvent(d2h_, kernels_done_[p], 0);
    cudaMemcpyAsync(slots_[slot].loss_pin, snap != nullptr ? snap : cfg_.loss_acc, 2 * sizeof(float), cudaMemcpyDeviceToHost, d2h_);
    cudaEventRecord(slots_[slot].done, d2h_);
    if (snap != nullptr) cudaEventRecord(loss_read_[p], d2h_);
    in_flight_.push_back({slot, slot, false});
    ++issued_;
    ++done;
    ++stats_.single_steps;
  }
  return done;
}

}  // namespace b2
