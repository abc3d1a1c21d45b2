// Native step executor -- see executor.cpp.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <deque>
#include <string>
#include <vector>

#include "loader.h"

namespace b2 {

struct StepConfig {
  float* params;
  float* momentum;
  float* grads_local;                // this rank's gradient bucket(s)
  void* grad_ptrs[8];                // every rank's bucket (symmetric mapping), [0] only when world == 1
  uint32_t* sig_ptrs[8];
  unsigned long long* step_counter;
  unsigned int* done_counter;
  float* loss_acc;                   // [2]
  unsigned char* in_dev[96];         // device input blocks, same layout as a loader slot: [x | pad | y]; [0..1] double-buffer
                                     // the per-step path, [g*chunk .. g*chunk+chunk) are the blocks of chunk group g (0/1);
                                     // [ring_base + slot] (when ring_base > 0): one block per loader slot for the per-step path
  int ring_base;                     // 0: per-step path double-buffers blocks 0/1; > 0: per-slot blocks start here
  float* loss_hist;                  // device [n blocks][2], same indexing as in_dev; originally [2*chunk][2]: cumulative loss as of each step of a chunk (written by the SGD kernel)
  int chunk;                         // steps per chunk (0/1 = per-step launches only), <= 8
  int B, x_u8, training, rank, world, cluster;
  unsigned long long seed;
  long long sample_base, grad_stride;
  float lr, mu, p_drop;
  float* aux;                        // conv2.weight in the kernels' smem layouts (maintained by the SGD kernel)
  void* inbox_ptrs[8];               // push exchange (sgd.cu): every rank's inbox
  int push;
  int wire_bf16;                     // push exchange: bf16 on the wire
  int fused_tail;                    // gradient exchange + SGD in the tail of the step kernel (one kernel per step)
  unsigned int* ticket;              // device scratch of the fused tail
  float* grad_slots;                 // one GPU, one CTA per sample: per-CTA slots [B][21888] and per-sample fc1 factors [B][384]
  float* factors;                    // of the step kernel, summed by reduce_sgd (sgd.cu) instead of red.add into the bucket
  unsigned int* flags;               // device [num_slots][2] zero-initialised words: {batch landed, loss snapshot written}
                                     // generations of the per-slot ring path's flag mode (nullptr: event mode)
};

class StepExecutor {
 public:
  StepExecutor(const StepConfig& cfg, NativeLoader* loader, int max_in_flight);
  ~StepExecutor();
  // Runs up to `max_steps` full-batch steps of the loader's current epoch.  Returns the number of steps done;
  // *pending_slot >= 0 (with *pending_count) if a short batch was fetched but not processed (caller handles it),
  // *epoch_done is set when the loader ran dry.
  int64_t run(int64_t max_steps, int* pending_slot, int64_t* pending_count, int* epoch_done);
  void drain();                      // wait for everything in flight, release loader slots
  bool prepare();                    // capture every graph of the hot loop now (keeps captures out of timed regions)
  double last_loss_cumulative() const { return last_loss_; }
  const std::string& error() const { return err_; }
  bool chunking() const { return chunk_ok_; }
  bool flag_mode() const { return flags_; }
  // host-side time accounting of run() (ns): where the feeding loop waits -- {loader next(), copy-event waits, loss retire
  // waits, everything else (driver calls)}, and the number of chunked / single steps issued
  struct Stats { long long next_ns = 0, copy_wait_ns = 0, retire_ns = 0, total_ns = 0, chunk_steps = 0, single_steps = 0; };
  const Stats& stats() const { return stats_; }
  void reset_stats() { stats_ = Stats(); }
  const std::string& chunk_note() const { return chunk_note_; }   // why chunk graphs were turned off (if they were)

 private:
  struct Slot {
    cudaEvent_t done = nullptr;      // loss of the step fed from this slot has landed in loss_pin
    float* loss_pin = nullptr;
  };
  bool capture(int parity);
  bool capture_chunk(int g, int size_idx);
  void release_copied(bool block_for_one);
  void drain_copies();
  void record_step(const void* x, const long long* y, float* loss_snapshot = nullptr, const unsigned int* in_flag = nullptr,
                   unsigned int* snap_flag = nullptr, unsigned int gen = 0);
  void retire_oldest();
  StepConfig cfg_;
  NativeLoader* loader_;
  int max_in_flight_;
  cudaStream_t copy_ = nullptr, compute_ = nullptr, d2h_ = nullptr;
  cudaGraphExec_t exec_[2] = {nullptr, nullptr};     // the two kernels, reading in_dev[parity]
  cudaEvent_t copied_[2] = {nullptr, nullptr}, kernels_done_[2] = {nullptr, nullptr}, loss_read_[2] = {nullptr, nullptr};
  bool direct_ = true;                               // per-step path: plain PDL stream launches instead of a graph per step
  bool flags_ = false;                               // per-slot ring path without cross-stream events (stream memory ops)
  std::vector<Slot> slots_;
  // chunk pipeline: K consecutive steps = three graph launches on three streams (see executor.cpp).  The slot of batch b is
  // b % num_slots, so the pinned addresses of a slot group are fixed; g = chunk parity selects the device block group.
  // kernels of k consecutive steps reading device blocks g*K .. g*K+k-1, for k = K, K/2, K/4, ... (index 0..3): a run of n
  // steps is issued as chunks of decreasing size, so only a short tail BATCH ever takes the per-step path
  cudaGraphExec_t comp_exec_[2][4] = {{nullptr, nullptr, nullptr, nullptr}, {nullptr, nullptr, nullptr, nullptr}};
  int chunk_sizes_[4] = {0, 0, 0, 0};
  int n_sizes_ = 0;
  std::vector<cudaEvent_t> copy_ev_;                   // "H2D copies of chunk c are done" (ring)
  struct CopyFlight { int ev, count; };
  std::deque<CopyFlight> copy_q_;                      // chunks whose loader slots are still held
  int held_ = 0;
  cudaEvent_t h2d_done_[2] = {nullptr, nullptr}, comp_done_[2] = {nullptr, nullptr}, d2h_done_[2] = {nullptr, nullptr};
  int64_t chunks_issued_ = 0;
  bool chunk_ok_ = false;
  struct Flight { int slot, ev_slot; bool released_at_copy; };
  std::deque<Flight> in_flight_;
  int64_t issued_ = 0;
  double last_loss_ = 0.0;
  std::string err_, chunk_note_;
  Stats stats_;
};

}  // namespace b2
