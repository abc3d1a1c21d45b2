// Native step executor: the training hot loop without the Python interpreter.
//
// The reference's hot loop (train_dist.py:115-124) is Python: DataLoader iteration, five framework calls and an
// optimizer step per batch.  Here the loop that feeds the GPU is C++ and software-pipelined over three streams:
//
//   copy stream    : ONE cudaMemcpyAsync per step -- the pinned loader slot [x | y] -> the slot's device input block
//   compute stream : waits for that copy, then the step's 2 kernels (convnet_step + allreduce_sgd / reduce_sgd) as plain
//                    stream launches with the programmatic-dependent-launch attribute: consecutive steps chain on the
//                    device as inside one long graph
//   d2h stream     : waits for the kernels, then copies the step's loss snapshot to the slot's pinned word; its event
//                    retires the step
//
// so the H2D copy of step i+1 and the loss read-back of step i-1 overlap the kernels of step i: 9 driver calls per step.
// Every loader slot has its own device block and loss snapshot, and a slot is rewritten only after the step that used it
// has retired (a retired step hands its slot back to the prefetch thread, loader.cpp), so no device-side "buffer free"
// event is needed.  At most `max_in_flight` steps are outstanding.  The GIL is released around run().
#include "executor.h"

#include <chrono>
#include <cstring>

extern "C" {
int b2_convnet_step_launch(const float* params, float* grads, const void* x, int x_u8, const long long* target,
                           float* loss_acc, float* out_logp, float* mask_out, const unsigned long long* step,
                           unsigned long long seed, long long sample_base, int B, int training, int backward,
                           float inv_bsz, float p_drop, int max_ctas, long long grad_stride, const float* aux,
                           float* det_partials, float* factors, int input_ready, cudaStream_t stream);
struct PeerPtrsC { void* p[8]; };
struct SignalPadsC { uint32_t* pad[8]; };
int b2_allreduce_sgd_launch(const PeerPtrsC* grads, const SignalPadsC* sig, float* params, float* momentum,
                            unsigned long long* step, size_t n_elems, float lr, float mu, float scale, int rank,
                            int world, int zero_grads, long long grad_stride, unsigned int* done_counter, float* aux,
                            const PeerPtrsC* inbox, const float* loss_acc, float* loss_snapshot, int wire_bf16,
                            const b2::LrSchedule* sched, float wd, int nesterov, float max_norm, float* clip_ws,
                            float* grad_norm_out, cudaStream_t stream);
int b2_reduce_sgd_launch(float* params, float* momentum, unsigned long long* step, unsigned int* done_counter, float lr, float mu,
                         float* aux, float* loss_acc, float* loss_snapshot, const float* slots, int n_slots, const float* factors,
                         int n_samples, float* grads, long long grad_stride, const b2::LrSchedule* sched, float wd, int nesterov,
                         float max_norm, float* clip_ws, float* grad_norm_out, int n_cta, cudaStream_t stream);
int b2_convnet_cluster_launch(const float* params, float* grads, const void* x, int x_u8, const long long* target,
                              float* loss_acc, float* out_logp, float* mask_out, const unsigned long long* step,
                              unsigned long long seed, long long sample_base, int B, int training, int backward,
                              float inv_bsz, float p_drop, int cluster, int max_clusters, long long grad_stride,
                              const float* aux, float* det_partials, cudaStream_t stream);
int b2_convnet_npar();
}

namespace b2 {

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
  for (int p = 0; p < 2; ++p) {
    if (copied_[p]) cudaEventDestroy(copied_[p]);
    if (kernels_done_[p]) cudaEventDestroy(kernels_done_[p]);
  }
  if (copy_) cudaStreamDestroy(copy_);
  if (compute_) cudaStreamDestroy(compute_);
  if (d2h_) cudaStreamDestroy(d2h_);
}

// Enqueues the two kernels of one step on the compute stream.
void StepExecutor::record_step(const void* x, const long long* y, float* loss_snapshot) {
  // one GPU, one CTA per sample: plain stores to the slots / factors, reduced in a fixed order by the optimizer kernel
  const bool slots = cfg_.grad_slots != nullptr && cfg_.world == 1 && cfg_.cluster <= 1;
  int rc = cfg_.cluster > 1
               ? b2_convnet_cluster_launch(cfg_.params, cfg_.grads_local, x, cfg_.x_u8, y, cfg_.loss_acc, nullptr, nullptr,
                                           cfg_.step_counter, cfg_.seed, cfg_.sample_base, cfg_.B, cfg_.training, 1,
                                           1.f / cfg_.B, cfg_.p_drop, cfg_.cluster, 0, cfg_.grad_stride, cfg_.aux, nullptr, compute_)
               : b2_convnet_step_launch(cfg_.params, cfg_.grads_local, x, cfg_.x_u8, y, cfg_.loss_acc, nullptr, nullptr,
                                        cfg_.step_counter, cfg_.seed, cfg_.sample_base, cfg_.B, cfg_.training, 1, 1.f / cfg_.B,
                                        cfg_.p_drop, 0, cfg_.grad_stride, cfg_.aux, slots ? cfg_.grad_slots : nullptr,
                                        slots ? cfg_.factors : nullptr, /*input_ready=*/1, compute_);
  int rc2 = 0;
  if (slots) {
    rc2 = b2_reduce_sgd_launch(cfg_.params, cfg_.momentum, cfg_.step_counter, cfg_.done_counter, cfg_.lr, cfg_.mu, cfg_.aux,
                               cfg_.loss_acc, loss_snapshot, cfg_.grad_slots, cfg_.B, cfg_.factors, cfg_.B, cfg_.grads_local,
                               cfg_.grad_stride, &cfg_.sched, cfg_.wd, cfg_.nesterov, cfg_.max_norm, cfg_.clip_ws, cfg_.grad_norm,
                               /*n_cta=*/0, compute_);
  } else {
    PeerPtrsC g;
    SignalPadsC sg;
    std::memcpy(g.p, cfg_.grad_ptrs, sizeof(g.p));
    std::memcpy(sg.pad, cfg_.sig_ptrs, sizeof(sg.pad));
    PeerPtrsC ib;
    std::memcpy(ib.p, cfg_.inbox_ptrs, sizeof(ib.p));
    rc2 = b2_allreduce_sgd_launch(&g, &sg, cfg_.params, cfg_.momentum, cfg_.step_counter, (size_t)b2_convnet_npar(),
                                  cfg_.lr, cfg_.mu, 1.f / cfg_.world, cfg_.rank, cfg_.world, 1, cfg_.grad_stride,
                                  cfg_.done_counter, cfg_.aux, cfg_.push ? &ib : nullptr, cfg_.loss_acc, loss_snapshot, cfg_.wire_bf16,
                                  &cfg_.sched, cfg_.wd, cfg_.nesterov, cfg_.max_norm, cfg_.clip_ws, cfg_.grad_norm, compute_);
  }
  if ((rc != 0 || rc2 != 0) && err_.empty())
    err_ = std::string("kernel launch failed: ") + cudaGetErrorString((cudaError_t)(rc ? rc : rc2));
}

void StepExecutor::retire_oldest() {
  const int s = in_flight_.front();
  in_flight_.pop_front();
  const long long t0 = now_ns();
  cudaEventSynchronize(slots_[s].done);
  stats_.retire_ns += now_ns() - t0;
  last_loss_ = (double)slots_[s].loss_pin[0];      // host read of this step's D2H loss copy
  loader_->release();
}

// A step retires after its loss D2H, which is ordered behind both of its kernels: once nothing is in flight, the
// kernels are done too.
void StepExecutor::drain() {
  while (!in_flight_.empty()) retire_oldest();
}

int64_t StepExecutor::run(int64_t max_steps, int* pending_slot, int64_t* pending_count, int* epoch_done) {
  *pending_slot = -1;
  *pending_count = 0;
  *epoch_done = 0;
  int64_t done = 0;
  struct Total { long long t0; Stats* s; ~Total() { s->total_ns += now_ns() - t0; } } total{now_ns(), &stats_};
  while (max_steps < 0 || done < max_steps) {
    while ((int)in_flight_.size() >= max_in_flight_) retire_oldest();
    int64_t count = 0;
    const long long tn = now_ns();
    const int slot = loader_->next(&count);
    stats_.next_ns += now_ns() - tn;
    if (slot < 0) { *epoch_done = 1; break; }
    if (count != cfg_.B) {            // short tail batch: give it back to the caller (eager path)
      drain();
      cudaStreamSynchronize(compute_);
      *pending_slot = slot;
      *pending_count = count;
      break;
    }
    // the slot's block and loss snapshot are free: the step that last used them retired before the slot was released
    const int p = (int)(issued_ & 1);
    unsigned char* blk = cfg_.in_dev + (size_t)slot * cfg_.in_stride;
    float* snap = cfg_.loss_hist + 2 * slot;
    cudaMemcpyAsync(blk, loader_->slot(slot).x, loader_->block_bytes(), cudaMemcpyHostToDevice, copy_);
    cudaEventRecord(copied_[p], copy_);
    cudaStreamWaitEvent(compute_, copied_[p], 0);
    err_.clear();
    record_step(blk, reinterpret_cast<const long long*>(blk + loader_->y_offset()), snap);
    if (!err_.empty()) return -1;
    cudaEventRecord(kernels_done_[p], compute_);
    // loss read-back: the cumulative loss as of THIS step (snapshotted on the device by the step's optimizer kernel)
    cudaStreamWaitEvent(d2h_, kernels_done_[p], 0);
    cudaMemcpyAsync(slots_[slot].loss_pin, snap, 2 * sizeof(float), cudaMemcpyDeviceToHost, d2h_);
    cudaEventRecord(slots_[slot].done, d2h_);
    in_flight_.push_back(slot);
    ++issued_;
    ++done;
    ++stats_.steps;
  }
  return done;
}

}  // namespace b2
