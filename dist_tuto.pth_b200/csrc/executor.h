// Native step executor -- see executor.cpp.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <deque>
#include <string>
#include <vector>

#include "loader.h"
#include "lr_schedule.h"

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
  unsigned char* in_dev;             // device input blocks, same layout as a loader slot: [x | pad | y]; block s (at
  size_t in_stride;                  // in_dev + s * in_stride) is fed from loader slot s
  float* loss_hist;                  // device [num_slots][2]: the cumulative loss as of the step fed from slot s (written by the SGD kernel)
  int B, x_u8, training, rank, world, cluster;
  unsigned long long seed;
  long long sample_base, grad_stride;
  float lr, mu, p_drop;
  float* aux;                        // conv2.weight in the kernels' smem layouts (maintained by the SGD kernel)
  void* inbox_ptrs[8];               // push exchange (sgd.cu): every rank's inbox
  int push;
  int wire_bf16;                     // push exchange: bf16 on the wire
  float* grad_slots;                 // one GPU, one CTA per sample: per-CTA slots [B][21888] and per-sample fc1 factors [B][384]
  float* factors;                    // of the step kernel, summed by reduce_sgd (sgd.cu) instead of red.add into the bucket
  LrSchedule sched;                  // lr schedule of every step's update (zero: constant lr)
};

class StepExecutor {
 public:
  StepExecutor(const StepConfig& cfg, NativeLoader* loader, int max_in_flight);
  ~StepExecutor();
  // Runs up to `max_steps` full-batch steps of the loader's current epoch.  Returns the number of steps done;
  // *pending_slot >= 0 (with *pending_count) if a short batch was fetched but not processed (caller handles it),
  // *epoch_done is set when the loader ran dry.
  int64_t run(int64_t max_steps, int* pending_slot, int64_t* pending_count, int* epoch_done);
  void drain();                      // retire every step in flight, release their loader slots
  double last_loss_cumulative() const { return last_loss_; }
  const std::string& error() const { return err_; }
  // host-side time accounting of run() (ns): where the feeding loop waits -- {loader next(), loss retire waits, everything
  // else (driver calls)}, and the number of steps issued
  struct Stats { long long next_ns = 0, retire_ns = 0, total_ns = 0, steps = 0; };
  const Stats& stats() const { return stats_; }
  void reset_stats() { stats_ = Stats(); }

 private:
  struct Slot {
    cudaEvent_t done = nullptr;      // loss of the step fed from this slot has landed in loss_pin
    float* loss_pin = nullptr;
  };
  void record_step(const void* x, const long long* y, float* loss_snapshot);
  void retire_oldest();
  StepConfig cfg_;
  NativeLoader* loader_;
  int max_in_flight_;
  cudaStream_t copy_ = nullptr, compute_ = nullptr, d2h_ = nullptr;
  cudaEvent_t copied_[2] = {nullptr, nullptr}, kernels_done_[2] = {nullptr, nullptr};
  std::vector<Slot> slots_;
  std::deque<int> in_flight_;        // loader slots of the steps issued and not retired yet, oldest first
  int64_t issued_ = 0;
  double last_loss_ = 0.0;
  std::string err_;
  Stats stats_;
};

}  // namespace b2
