// Python bindings (pybind11 / torch extension) for the native runtime and the sm_90a kernels.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "adafactor.h"
#include "adamw.h"
#include "ema.h"
#include "executor.h"
#include "flat_scalars.h"
#include "batchnorm.h"
#include "layerwise.h"
#include "loader.h"
#include "param_groups.h"
#include "rmsprop.h"

#define B2_MAX_RANKS 8
struct PeerPtrs { void* p[B2_MAX_RANKS]; };
struct SignalPadsH { uint32_t* pad[B2_MAX_RANKS]; };

extern "C" {
const char* b2_symm_last_error();
int b2_symm_caps(int dev, int* caps);
int b2_symm_granularity(int dev, int ndev, int want_multicast, size_t* gran);
int b2_symm_create(int dev, size_t bytes, unsigned long long* handle, int* fd);
int b2_symm_import(int fd, unsigned long long* handle);
int b2_symm_map(int dev, unsigned long long handle, size_t bytes, size_t align, unsigned long long* ptr);
int b2_symm_unmap(unsigned long long ptr, size_t bytes);
int b2_symm_release(unsigned long long handle);
int b2_mc_create(int ndev, size_t bytes, unsigned long long* handle, int* fd);
int b2_mc_add_device(unsigned long long mc, int dev);
int b2_mc_bind(unsigned long long mc, unsigned long long mem, size_t bytes);
int b2_mc_unbind(unsigned long long mc, int dev, size_t bytes);
int b2_ipc_alloc(size_t bytes, unsigned long long* ptr, unsigned char* handle64);
int b2_ipc_open(const unsigned char* handle64, unsigned long long* ptr);
int b2_ipc_close(unsigned long long ptr);
int b2_ipc_free(unsigned long long ptr);

int b2_allreduce_launch(int variant, int bf16, const PeerPtrs* bufs, const SignalPadsH* sig, void* mc, const void* src,
                        int src_f32, void* dst, int dst_f32, size_t n_vec, float scale, int rank, int world,
                        int max_blocks, const PeerPtrs* inbox, size_t ll_cap, int op, int root, cudaStream_t stream);
int b2_allreduce_dtype_launch(int variant, int dtype, const PeerPtrs* bufs, const SignalPadsH* sig, void* mc, const void* src,
                              int src_f32, void* dst, int dst_f32, size_t n_vec, float scale, int rank, int world,
                              int max_blocks, const PeerPtrs* inbox, size_t ll_cap, int op, int root, cudaStream_t stream);
int b2_reduce_scatter_launch(int variant, int dtype, int op, const PeerPtrs* bufs, const SignalPadsH* sig, const void* src,
                             void* dst, size_t n_vec, int rank, int world, int max_blocks, const PeerPtrs* inbox,
                             size_t ll_cap, cudaStream_t stream);
int b2_alltoall_launch(int variant, const PeerPtrs* bufs, const SignalPadsH* sig, const void* src, void* dst, size_t n_vec,
                       int rank, int world, int max_blocks, const PeerPtrs* inbox, size_t ll_cap, cudaStream_t stream);
void b2_alltoallv_config(size_t* chunk, size_t* header);
int b2_alltoallv_launch(const PeerPtrs* bufs, const SignalPadsH* sig, const void* const* src, const unsigned long long* src_bytes,
                        void* const* dst, const unsigned long long* dst_bytes, int rank, int world, int max_blocks,
                        cudaStream_t stream);
int b2_barrier_launch(const SignalPadsH* sig, int rank, int world, cudaStream_t stream);
void b2_p2p_config(int* ctas, int* slots, size_t* chunk, int* pad_words);
int b2_p2p_send_launch(const PeerPtrs* box, const SignalPadsH* sig, const void* src, size_t nbytes, int rank, int peer,
                       int world, cudaStream_t stream);
int b2_p2p_recv_launch(const PeerPtrs* box, const SignalPadsH* sig, void* dst, size_t nbytes, int rank, int peer,
                       int world, cudaStream_t stream);
int b2_p2p_batch_capacity();
int b2_p2p_batch_launch(const PeerPtrs* box, const SignalPadsH* sig, const int* send, const int* peer, void* const* msg,
                        const size_t* nbytes, int n_ops, int rank, int world, cudaStream_t stream);
int b2_allreduce_sgd_launch(const PeerPtrs* grads, const SignalPadsH* sig, float* params, float* momentum,
                            unsigned long long* step, size_t n_elems, float lr, float mu, float scale, int rank,
                            int world, int zero_grads, long long grad_stride, unsigned int* done_counter, float* aux,
                            const PeerPtrs* inbox, const float* loss_acc, float* loss_snapshot, int wire_bf16,
                            const b2::LrSchedule* sched, float wd, int nesterov, float max_norm, float* clip_ws,
                            float* grad_norm_out, cudaStream_t stream);
int b2_lr_schedule_eval_launch(const b2::LrSchedule* sched, float base, const long long* steps, float* out, long long n,
                               cudaStream_t stream);
int b2_sgd_flat_launch(float* p, float* m, const float* g, size_t n, float lr, float mu, float wd, int zero_grad, int nesterov,
                       float max_norm, const double* sqnorms, int n_buckets, float* grad_norm_out, const float* grad_scale,
                       cudaStream_t stream);
int b2_sharded_sgd_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const SignalPadsH* sig, float* momentum,
                          size_t n_vec, float lr, float mu, float wd, int nesterov, float scale, int zero_grad, int rank,
                          int world, int max_blocks, cudaStream_t stream);
int b2_adamw_flat_launch(float* p, float* m, float* v, float* g, size_t n, const b2::AdamwScalars* s, int zero_grad,
                         float max_norm, const double* sqnorms, int n_buckets, float* grad_norm_out, const float* grad_scale,
                         cudaStream_t stream);
int b2_sharded_adamw_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const SignalPadsH* sig, float* exp_avg,
                            float* exp_avg_sq, size_t n_vec, const b2::AdamwScalars* s, float scale, int zero_grad, int rank,
                            int world, int max_blocks, cudaStream_t stream);
int b2_sgd_flat_grouped_launch(float* p, float* m, const float* g, size_t n, const uint8_t* map, const b2::SgdGroups* gs,
                               int n_groups, float mu, int zero_grad, int nesterov, float max_norm, const double* sqnorms,
                               int n_buckets, float* grad_norm_out, const float* grad_scale, cudaStream_t stream);
int b2_adamw_flat_grouped_launch(float* p, float* m, float* v, float* g, size_t n, const uint8_t* map, const b2::AdamwScalars* s,
                                 const b2::AdamwGroups* gs, int n_groups, int zero_grad, float max_norm, const double* sqnorms,
                                 int n_buckets, float* grad_norm_out, const float* grad_scale, cudaStream_t stream);
int b2_sharded_sgd_grouped_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const SignalPadsH* sig,
                                  float* momentum, const uint8_t* map, const b2::SgdGroups* gs, int n_groups, size_t n_vec, float mu,
                                  int nesterov, float scale, int zero_grad, int rank, int world, int max_blocks,
                                  cudaStream_t stream);
int b2_sharded_adamw_grouped_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const SignalPadsH* sig,
                                    float* exp_avg, float* exp_avg_sq, const uint8_t* map, const b2::AdamwScalars* s,
                                    const b2::AdamwGroups* gs, int n_groups, size_t n_vec, float scale, int zero_grad, int rank,
                                    int world, int max_blocks, cudaStream_t stream);
int b2_layerwise_launch(int lamb, const b2::LwArgs* a, cudaStream_t stream);
int b2_sharded_layerwise_launch(int lamb, int bf16, const PeerPtrs* grads, const PeerPtrs* params, const PeerPtrs* sums,
                                const SignalPadsH* sig, const b2::LwArgs* lw, size_t n_vec, float scale, int rank, int world,
                                int max_blocks, cudaStream_t stream);
int b2_adafactor_launch(const b2::AfArgs* a, cudaStream_t stream);
int b2_flat_scalars_launch(const b2::FlatHyper* table, unsigned long long* counter, b2::FlatScalars* block, int advance,
                           const float* found_inf, cudaStream_t stream);
int b2_sgd_flat_cap_launch(float* p, float* m, const float* g, size_t n, const uint8_t* map, const b2::FlatScalars* blk, float mu,
                           int zero_grad, int nesterov, float max_norm, const double* sqnorms, int n_buckets, float* grad_norm_out,
                           const float* grad_scale, const float* found_inf, cudaStream_t stream);
int b2_adamw_flat_cap_launch(float* p, float* m, float* v, float* g, size_t n, const uint8_t* map, const b2::FlatScalars* blk,
                             int zero_grad, float max_norm, const double* sqnorms, int n_buckets, float* grad_norm_out,
                             const float* grad_scale, const float* found_inf, cudaStream_t stream);
int b2_sharded_sgd_cap_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const SignalPadsH* sig, float* momentum,
                              const uint8_t* map, const b2::FlatScalars* blk, size_t n_vec, float mu, int nesterov, float scale,
                              int zero_grad, int rank, int world, int max_blocks, cudaStream_t stream);
int b2_sharded_adamw_cap_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const SignalPadsH* sig, float* exp_avg,
                                float* exp_avg_sq, const uint8_t* map, const b2::FlatScalars* blk, size_t n_vec, float scale,
                                int zero_grad, int rank, int world, int max_blocks, cudaStream_t stream);
int b2_rmsprop_flat_launch(float* p, float* sq, float* ga, float* buf, float* g, size_t n, const uint8_t* map,
                           const b2::RmspropScalars* s, const b2::SgdGroups* gs, int n_groups, const b2::FlatScalars* blk,
                           int zero_grad, float max_norm, const double* sqnorms, int n_buckets, float* grad_norm_out,
                           const float* grad_scale, const float* found_inf, cudaStream_t stream);
int b2_sharded_rmsprop_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const SignalPadsH* sig, float* square_avg,
                              float* grad_avg, float* momentum_buffer, const uint8_t* map, const b2::RmspropScalars* s,
                              const b2::SgdGroups* gs, int n_groups, size_t n_vec, float scale, int zero_grad, int rank, int world,
                              int max_blocks, cudaStream_t stream);
int b2_sharded_rmsprop_cap_launch(int bf16, const PeerPtrs* grads, const PeerPtrs* params, const SignalPadsH* sig,
                                  float* square_avg, float* grad_avg, float* momentum_buffer, const uint8_t* map,
                                  const b2::FlatScalars* blk, const b2::RmspropScalars* s, size_t n_vec, float scale, int zero_grad,
                                  int rank, int world, int max_blocks, cudaStream_t stream);
int b2_ema_launch(const b2::EmaEntry* table, int n_entries, long long n_vec, long long n_scalar, float w, int mode,
                  const long long* counter, long long every, long long warmup, cudaStream_t stream);
int b2_grad_sqnorm_ws_floats();
int b2_grad_sqnorm_launch(const float* g, size_t n, float* ws, double* sqnorms, int k, const float* grad_scale,
                          cudaStream_t stream);
size_t b2_clip_ws_floats(size_t n_elems);
int b2_bn_launch(int kind, int dtype, int vec, int cl, long long M, long long L, int max_blocks, const b2::bn::Args* args,
                 unsigned int* grid_out, cudaStream_t stream);
size_t b2_convnet_smem_bytes();
int b2_convnet_npar();
int b2_convnet_step_launch(const float* params, float* grads, const void* x, int x_u8, const long long* target,
                           float* loss_acc, float* out_logp, float* mask_out, const unsigned long long* step,
                           unsigned long long seed, long long sample_base, int B, int training, int backward,
                           float inv_bsz, float p_drop, int max_ctas, long long grad_stride, const float* aux,
                           float* det_partials, float* factors, int input_ready, cudaStream_t stream);
int b2_reduce_sgd_launch(float* params, float* momentum, unsigned long long* step, unsigned int* done_counter, float lr, float mu,
                         float* aux, float* loss_acc, float* loss_snapshot, const float* slots, int n_slots, const float* factors,
                         int n_samples, float* grads, long long grad_stride, const b2::LrSchedule* sched, float wd, int nesterov,
                         float max_norm, float* clip_ws, float* grad_norm_out, int n_cta, cudaStream_t stream);
int b2_reduce_units();
int b2_convnet_eval_max_ctas(int dev);
int b2_convnet_eval_samples_per_cta();
int b2_convnet_eval_launch(const float* params, const void* x, int x_u8, const long long* target, double* result, int* slots,
                           float* out_logp, long long N, float mean, float std, int dev, cudaStream_t stream);
void b2_set_phase_ts(unsigned long long* p);
int b2_det_reduce_launch(const float* partials, int n_slots, long long slot_stride, float* grads, const unsigned long long* step,
                         long long grad_stride, size_t n_elems, float* loss_acc, cudaStream_t stream);
int b2_convnet_cluster_launch(const float* params, float* grads, const void* x, int x_u8, const long long* target,
                              float* loss_acc, float* out_logp, float* mask_out, const unsigned long long* step,
                              unsigned long long seed, long long sample_base, int B, int training, int backward,
                              float inv_bsz, float p_drop, int cluster, int max_clusters, long long grad_stride,
                              const float* aux, float* det_partials, cudaStream_t stream);
int b2_gemm_available();
int b2_gemm_bf16_launch(const void* a, const void* b, void* c, const float* bias, int M, int N, int K, int relu,
                        int out_bf16, cudaStream_t stream);
const char* b2_gemm_last_error();
struct BtBuffers {
  void *P1, *P2, *H, *DH, *dP2, *DC, *W2K, *W2R, *W3K, *W3T;
  unsigned char *A1, *A2;
  float *Hrelu, *DLOG, *G1, *B3P;
};
const char* b2_bt_last_error();
int b2_bt_pack_weights(const float* params, const BtBuffers* bf, cudaStream_t stream);
int b2_bt_step_launch(const float* params, float* grads, const void* x, int x_u8, const long long* target, const BtBuffers* bf,
                      float* loss_acc, float* out_logp, const unsigned long long* step, unsigned long long seed,
                      long long sample_base, int B, int training, int backward, float inv_bsz, float p_drop, int stage_mask,
                      cudaStream_t stream);
const char* b2_probe_last_error();
int b2_tma_probe(const void* tensor, int rank, const unsigned long long* dims, const unsigned long long* strides_bytes,
                 const unsigned int* box, int swizzle, const int* coords, unsigned int bytes, unsigned char* out,
                 cudaStream_t stream);
int b2_wgmma_probe(const unsigned char* a_img, unsigned int a_bytes, const unsigned char* b_img, unsigned int b_bytes,
                   int a_mn, const unsigned long long* ops, int n_ops, int n, float* dump, cudaStream_t stream);
}

namespace {

void ck_symm(int rc, const char* what) {
  if (rc != 0) throw std::runtime_error(std::string(what) + " failed (rc=" + std::to_string(rc) + "): " + b2_symm_last_error());
}
void ck_cuda(int rc, const char* what) {
  if (rc != 0) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString((cudaError_t)rc));
}
cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

PeerPtrs to_ptrs(const std::vector<unsigned long long>& v) {
  TORCH_CHECK(v.size() <= B2_MAX_RANKS, "at most 8 ranks per symmetric world");
  PeerPtrs p;
  for (int i = 0; i < B2_MAX_RANKS; ++i) p.p[i] = i < (int)v.size() ? (void*)(uintptr_t)v[i] : nullptr;
  return p;
}
SignalPadsH to_sig(const std::vector<unsigned long long>& v) {
  TORCH_CHECK(v.size() <= B2_MAX_RANKS, "at most 8 ranks per symmetric world");
  SignalPadsH s;
  for (int i = 0; i < B2_MAX_RANKS; ++i) s.pad[i] = i < (int)v.size() ? (uint32_t*)(uintptr_t)v[i] : nullptr;
  return s;
}

// The comm kernels index their per-rank pointer lists by rank: a missing entry would be a null device pointer.
void check_world(int rank, int world, const char* what) {
  TORCH_CHECK(world >= 1 && world <= B2_MAX_RANKS, what, ": world must be in 1..8, got ", world);
  TORCH_CHECK(rank >= 0 && rank < world, what, ": rank ", rank, " is outside [0, ", world, ")");
}

void check_cuda_contig(const torch::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.is_contiguous(), name, " must be a contiguous CUDA tensor");
}

// An lr schedule from its plain-tuple form (ops/optim.LRSchedule.as_tuple):
//   (kind, warmup, total, start, gamma, min_factor, milestones); None -> no schedule (the lr as given)
// torch.optim.SGD's rules for weight decay and Nesterov momentum (dampening is always 0 here)
void check_sgd_options(double weight_decay, bool nesterov, double mu, const char* what) {
  TORCH_CHECK(weight_decay >= 0.0, what, ": weight_decay must be >= 0, got ", weight_decay);
  TORCH_CHECK(!nesterov || mu != 0.0, what, ": nesterov needs a nonzero momentum");
}

// torch.nn.utils.clip_grad_norm_'s max_norm (norm type 2): None (no clipping) or a finite value > 0.  Returns the value the
// launchers take, 0 for None.
float check_max_grad_norm(const py::object& o, const char* what) {
  if (o.is_none()) return 0.f;
  const double c = o.cast<double>();
  TORCH_CHECK(std::isfinite(c) && c > 0.0 && (float)c > 0.f && std::isfinite((float)c), what,
              ": max_grad_norm must be None or a finite value > 0, got ", c);
  return (float)c;
}

// The clip instances' workspace for `n` flat elements: fp32 CUDA, b2_clip_ws_floats(n) floats, zero before its first use.
float* clip_ws_ptr(float max_norm, const c10::optional<torch::Tensor>& ws, int64_t n, const char* what) {
  if (max_norm == 0.f) return nullptr;
  TORCH_CHECK(ws.has_value() && ws->is_cuda() && ws->is_contiguous() && ws->scalar_type() == torch::kFloat32 &&
              ws->numel() >= (int64_t)b2_clip_ws_floats((size_t)n) && (uintptr_t)ws->data_ptr() % 16 == 0, what,
              ": max_grad_norm needs clip_workspace, a 16-byte aligned fp32 CUDA tensor of clip_workspace_numel(", n, ") = ",
              b2_clip_ws_floats((size_t)n), " elements");
  return ws->data_ptr<float>();
}
float* grad_norm_ptr(const c10::optional<torch::Tensor>& t, const char* what) {
  if (!t.has_value()) return nullptr;
  TORCH_CHECK(t->is_cuda() && t->scalar_type() == torch::kFloat32 && t->numel() >= 1, what, ": grad_norm_out: fp32 CUDA [1]");
  return t->data_ptr<float>();
}
// GradScaler's grad_scale or found_inf (fp16 loss scaling, csrc/sgd_device.cuh): an fp32 CUDA scalar on the device of `like`,
// or null when absent
const float* amp_scalar_ptr(const c10::optional<torch::Tensor>& t, const torch::Tensor& like, const char* what, const char* name) {
  if (!t.has_value()) return nullptr;
  TORCH_CHECK(t->is_cuda() && t->device() == like.device() && t->scalar_type() == torch::kFloat32 && t->numel() == 1, what, ": ",
              name, ": an fp32 CUDA tensor of one element on the device of the buffers");
  return t->data_ptr<float>();
}
// GradScaler's (grad_scale, found_inf) of an update launch (see amp_scalar_ptr).  A capturable update (`paired`) decides the
// skip on the device, so it takes grad_scale only with found_inf.
std::pair<const float*, const float*> amp_pair(const c10::optional<torch::Tensor>& grad_scale,
                                               const c10::optional<torch::Tensor>& found_inf, bool paired, const torch::Tensor& like,
                                               const char* what) {
  TORCH_CHECK(!paired || found_inf.has_value() || !grad_scale.has_value(), what,
              ": grad_scale comes with found_inf (GradScaler sets both)");
  return {amp_scalar_ptr(grad_scale, like, what, "grad_scale"), amp_scalar_ptr(found_inf, like, what, "found_inf")};
}

// The clipping arguments of an update launch: max_norm (0 without clipping), grad_sqnorm's per-bucket sums and their count,
// and the optional grad_norm_out.
struct Clip {
  float max_norm;
  const double* sq;
  int n_buckets;
  float* gn;
};
Clip clip_args(const py::object& max_grad_norm, const c10::optional<torch::Tensor>& sqnorms,
               const c10::optional<torch::Tensor>& grad_norm_out, const char* what) {
  Clip c{check_max_grad_norm(max_grad_norm, what), nullptr, 0, nullptr};
  if (c.max_norm > 0.f) {
    TORCH_CHECK(sqnorms.has_value() && sqnorms->is_cuda() && sqnorms->is_contiguous() && sqnorms->scalar_type() == torch::kFloat64 &&
                sqnorms->numel() >= 1, what, ": max_grad_norm needs sqnorms, fp64 CUDA [buckets] from grad_sqnorm");
    c.sq = sqnorms->data_ptr<double>();
    c.n_buckets = (int)sqnorms->numel();
  }
  c.gn = grad_norm_ptr(grad_norm_out, what);
  return c;
}

// The flat buffers of an update (parameters, gradients, state; null entries are absent optional states): contiguous 16-byte
// aligned fp32 CUDA tensors on one device with `n` elements each (at_least: n or more).  `names` names them in the message.
// The first entry is never null.
void check_flats(const std::vector<const torch::Tensor*>& ts, int64_t n, bool at_least, const char* names, const char* what) {
  for (const torch::Tensor* t : ts)
    TORCH_CHECK(t == nullptr || (t->is_cuda() && t->is_contiguous() && t->scalar_type() == torch::kFloat32 &&
                                 t->device() == ts[0]->device() && (at_least ? t->numel() >= n : t->numel() == n) &&
                                 (uintptr_t)t->data_ptr() % 16 == 0),
                what, ": ", names, ": 16-byte aligned contiguous fp32 CUDA tensors on one device, of ",
                at_least ? "at least " : "one size, ", n, " elements");
}

// The per-rank pointers of a sharded update (csrc/sharded_sgd.cu, csrc/sharded_layerwise.cu): one gradient bucket,
// parameter flat, signal pad and, for the layer-wise kernels (`sums` given), sums buffer per rank, none null or misaligned,
// and a bucket of n_vec 16-byte vectors that splits into `world` slices.  `shard` is the elements of one slice.
struct Peers {
  int64_t shard;
  PeerPtrs grads, params, sums;
  SignalPadsH sigs;
};
Peers sharded_peers(const char* what, const std::vector<unsigned long long>& grads, const std::vector<unsigned long long>& params,
                    const std::vector<unsigned long long>* sums, const std::vector<unsigned long long>& sigs, size_t n_vec, bool bf16,
                    int rank, int world) {
  check_world(rank, world, what);
  TORCH_CHECK((int)grads.size() == world && (int)params.size() == world && (int)sigs.size() == world &&
              (sums == nullptr || (int)sums->size() == world), what, ": one gradient bucket, parameter flat, ",
              sums != nullptr ? "sums buffer " : "", "and signal pad per rank, got ", grads.size(), ", ", params.size(),
              sums != nullptr ? ", " + std::to_string(sums->size()) : "", " and ", sigs.size(), " for world ", world);
  TORCH_CHECK(n_vec % (size_t)world == 0, what, ": every rank owns n_vec / world vectors, so n_vec must be a multiple of world "
              "(pad the buffers), got n_vec ", n_vec, " for world ", world);
  for (const auto* v : {&grads, &params, &sigs, sums != nullptr ? sums : &sigs})
    for (unsigned long long q : *v) TORCH_CHECK(q != 0 && q % 16 == 0, what, ": null or misaligned per-rank pointer");
  return {(int64_t)(n_vec / (size_t)world * (bf16 ? 8 : 4)), to_ptrs(grads), to_ptrs(params),
          to_ptrs(sums != nullptr ? *sums : std::vector<unsigned long long>()), to_sig(sigs)};
}

// One AdamW update's scalars (csrc/adamw.h), computed by the host in fp64 (ops/optim.py adamw_scalars): (1 - lr*wd,
// 1 - beta1, beta2, 1 - beta2, lr / bc1, sqrt(bc2), eps), each rounded once to fp32 here.
b2::AdamwScalars to_adamw(const std::vector<double>& v, const char* what) {
  TORCH_CHECK(v.size() == 7, what, ": scalars: (decay, 1 - beta1, beta2, 1 - beta2, step_size, sqrt(bc2), eps), got ", v.size(),
              " values");
  for (double x : v) TORCH_CHECK(std::isfinite(x) && std::isfinite((float)x), what, ": scalars must be finite in fp32");
  TORCH_CHECK((float)v[5] > 0.f && v[6] >= 0.0, what, ": sqrt(bc2) must be > 0 (update t >= 1) and eps >= 0");
  b2::AdamwScalars a;
  a.decay = (float)v[0]; a.w1 = (float)v[1]; a.beta2 = (float)v[2]; a.c2 = (float)v[3];
  a.step_size = (float)v[4]; a.sbc2 = (float)v[5]; a.eps = (float)v[6];
  return a;
}

// One RMSprop update's scalars (csrc/rmsprop.h), computed by the host in fp64 (ops/optim.py rmsprop_scalars): (lr,
// weight_decay, alpha, 1 - alpha, eps, momentum), each rounded once to fp32 here.  `centered` and momentum > 0 say which
// optional states the update has.
b2::RmspropScalars to_rmsprop(const std::vector<double>& v, bool centered, const char* what) {
  TORCH_CHECK(v.size() == 6, what, ": scalars: (lr, weight_decay, alpha, 1 - alpha, eps, momentum), got ", v.size(), " values");
  for (double x : v) TORCH_CHECK(std::isfinite(x) && std::isfinite((float)x), what, ": scalars must be finite in fp32");
  TORCH_CHECK(v[1] >= 0.0 && v[2] >= 0.0 && v[4] >= 0.0 && v[5] >= 0.0, what,
              ": weight_decay, alpha, eps and momentum must be >= 0");
  b2::RmspropScalars s;
  s.lr = (float)v[0]; s.wd = (float)v[1]; s.alpha = (float)v[2]; s.c = (float)v[3]; s.eps = (float)v[4]; s.mu = (float)v[5];
  s.centered = centered ? 1 : 0;
  s.momentum = v[5] > 0.0 ? 1 : 0;
  return s;
}

// The state flats of an RMSprop update: square_avg, plus grad_avg exactly when centered and momentum_buffer exactly when
// momentum > 0, checked with the update's other flats `flats` (check_flats).  Returns the optional states' pointers, null
// when absent.
std::pair<float*, float*> rmsprop_state(std::vector<const torch::Tensor*> flats, const torch::Tensor& square_avg,
                                        const c10::optional<torch::Tensor>& grad_avg,
                                        const c10::optional<torch::Tensor>& momentum_buffer, const b2::RmspropScalars& s,
                                        int64_t n, bool at_least, const char* names, const char* what) {
  TORCH_CHECK(grad_avg.has_value() == (s.centered != 0), what, ": grad_avg is given exactly when centered=True");
  TORCH_CHECK(momentum_buffer.has_value() == (s.momentum != 0), what, ": momentum_buffer is given exactly when momentum > 0");
  flats.insert(flats.end(), {&square_avg, grad_avg.has_value() ? &*grad_avg : nullptr,
                             momentum_buffer.has_value() ? &*momentum_buffer : nullptr});
  check_flats(flats, n, at_least, names, what);
  return {grad_avg.has_value() ? grad_avg->data_ptr<float>() : nullptr,
          momentum_buffer.has_value() ? momentum_buffer->data_ptr<float>() : nullptr};
}

// Parameter groups (csrc/param_groups.h): the group map of `n_ids` parameter vectors (uint8 CUDA, 1..64 groups) and two
// per-group scalar lists of one length, rounded once to fp32.  Returns the number of groups.
int check_groups(const torch::Tensor& map, int64_t n_ids, const std::vector<double>& a, const std::vector<double>& b,
                 float* out_a, float* out_b, const char* what) {
  TORCH_CHECK(map.is_cuda() && map.is_contiguous() && map.scalar_type() == torch::kUInt8 && map.numel() >= n_ids, what,
              ": group_map: contiguous uint8 CUDA of at least ", n_ids, " ids (one per fp32 parameter vector)");
  TORCH_CHECK(!a.empty() && a.size() <= (size_t)b2::kMaxGroups && a.size() == b.size(), what, ": 1..", b2::kMaxGroups,
              " groups with one value of each per-group scalar, got ", a.size(), " and ", b.size());
  for (size_t i = 0; i < a.size(); ++i) {
    TORCH_CHECK(std::isfinite((float)a[i]) && std::isfinite((float)b[i]), what, ": per-group scalars must be finite in fp32");
    out_a[i] = (float)a[i];
    out_b[i] = (float)b[i];
  }
  return (int)a.size();
}

// FlatLAMB / FlatLARS (csrc/layerwise.cu, csrc/sharded_layerwise.cu): the chunk table (layerwise.h) of the elements [lo, hi)
// of one bucket of n elements, from its tensors' offsets, sizes and adapt flags, checked on the host and uploaded to `device`:
// each tensor's piece of [lo, hi) cut into chunks of at most kLwChunk elements from the piece's start, then one row per
// tensor of the bucket.  Returns (table, number of chunks); `what` names the binding in the messages.
std::pair<torch::Tensor, int64_t> lw_table(const std::vector<int64_t>& offsets, const std::vector<int64_t>& numels,
                                           const std::vector<bool>& adapt, int64_t n, int64_t lo, int64_t hi, torch::Device device,
                                           const char* what) {
  TORCH_CHECK(!offsets.empty() && offsets.size() == numels.size() && offsets.size() == adapt.size(),
              what, ": one offset, size and adapt flag per tensor, at least one tensor");
  TORCH_CHECK(offsets.size() < (size_t)INT32_MAX, what, ": too many tensors");
  std::vector<int64_t> chunks, tens;
  int64_t end = 0;
  for (size_t t = 0; t < offsets.size(); ++t) {
    const int64_t o = offsets[t], k = numels[t];
    TORCH_CHECK(o % 4 == 0 && k >= 0 && o >= end && o + k <= n, what, ": tensor ", t, " at [", o, ", ", o + k,
                ") must start at a multiple of 4 elements, after the previous tensor, inside the flat of ", n, " elements");
    end = o + k;
    tens.push_back((int64_t)chunks.size() / b2::kLwRow);
    int64_t c = 0;
    const int64_t a = std::max(o, lo), b = std::min(o + k, hi);
    for (int64_t s = a; s < b; s += b2::kLwChunk, ++c) {
      chunks.push_back(s);
      chunks.push_back(std::min<int64_t>(b2::kLwChunk, b - s));
      chunks.push_back((int64_t)t);
    }
    tens.push_back(c);
    tens.push_back(adapt[t] ? 1 : 0);
  }
  const int64_t n_chunks = (int64_t)chunks.size() / b2::kLwRow;
  chunks.insert(chunks.end(), tens.begin(), tens.end());
  auto host = torch::tensor(chunks, torch::dtype(torch::kInt64));
  return {host.to(device), n_chunks};
}

py::tuple layerwise_table(const std::vector<int64_t>& offsets, const std::vector<int64_t>& numels, const std::vector<bool>& adapt,
                          int64_t n, torch::Device device) {
  auto [table, n_chunks] = lw_table(offsets, numels, adapt, n, 0, n, device, "layerwise_table");
  TORCH_CHECK(n_chunks >= 1 && n_chunks < INT32_MAX, "layerwise_table: the tensors hold no element, or too many chunks");
  return py::make_tuple(table, n_chunks);
}

// The table of rank `rank`'s slice [rank * n / world, (rank + 1) * n / world) of a padded bucket of n elements (sharded
// FlatLAMB / FlatLARS).  A slice of padding only has no chunk; its tensor rows are still there.  The kernels index the state
// shards relative to the slice start, so the table keeps the slice it was built for, and the launch bindings refuse it for
// another rank, world size or bucket size.
struct ShardedLwTable {
  torch::Tensor table;    // int64 CUDA: n_chunks + tensors rows (layerwise.h)
  int64_t n_chunks, n;
  int rank, world;
};

ShardedLwTable sharded_layerwise_table(const std::vector<int64_t>& offsets, const std::vector<int64_t>& numels,
                                       const std::vector<bool>& adapt, int64_t n, int rank, int world, torch::Device device) {
  check_world(rank, world, "sharded_layerwise_table");
  TORCH_CHECK(n % (4 * (int64_t)world) == 0, "sharded_layerwise_table: the padded bucket of ", n, " elements must split into ", world,
              " slices of whole 16-byte vectors");
  const int64_t per = n / world;
  auto [table, n_chunks] = lw_table(offsets, numels, adapt, n, rank * per, (rank + 1) * per, device, "sharded_layerwise_table");
  TORCH_CHECK(n_chunks < INT32_MAX, "sharded_layerwise_table: too many chunks");
  return {table, n_chunks, n, rank, world};
}

// The arguments every layer-wise launch shares: the table, the workspaces and clipping.  `states` are the state flats.
b2::LwArgs layerwise_args(const char* what, torch::Tensor& p, torch::Tensor& g, const std::vector<torch::Tensor*>& states,
                          const torch::Tensor& table, int64_t n_chunks, torch::Tensor& partials, torch::Tensor& tickets,
                          torch::Tensor& sums, torch::Tensor& ratios, bool zero_grad, const py::object& max_grad_norm,
                          const c10::optional<torch::Tensor>& sqnorms, const c10::optional<torch::Tensor>& grad_norm_out,
                          const c10::optional<torch::Tensor>& grad_scale) {
  std::vector<const torch::Tensor*> flats = {&p, &g};
  flats.insert(flats.end(), states.begin(), states.end());
  check_flats(flats, p.numel(), false, "parameters, gradients and state", what);
  for (const torch::Tensor* t : {&table, (const torch::Tensor*)&partials, (const torch::Tensor*)&tickets,
                                 (const torch::Tensor*)&sums, (const torch::Tensor*)&ratios}) {
    check_cuda_contig(*t, what);
    TORCH_CHECK(t->device() == p.device(), what, ": the table and the workspaces live on the parameters' device");
  }
  const int64_t n_tensors = tickets.numel();
  TORCH_CHECK(n_chunks >= 1 && n_chunks <= p.numel() && n_tensors >= 1 && table.scalar_type() == torch::kInt64 &&
              table.numel() == (n_chunks + n_tensors) * b2::kLwRow, what, ": table: int64 of (chunks + tensors) * ", b2::kLwRow,
              " entries from layerwise_table, tickets: one per tensor");
  TORCH_CHECK(tickets.scalar_type() == torch::kInt32, what, ": tickets: int32 [tensors], zero before the first call");
  TORCH_CHECK(partials.scalar_type() == torch::kFloat32 && partials.numel() == 2 * n_chunks && (uintptr_t)partials.data_ptr() % 8 == 0,
              what, ": partials: fp32 [2 * chunks]");
  TORCH_CHECK(sums.scalar_type() == torch::kFloat64 && sums.numel() == 2 * n_tensors, what, ": sums: fp64 [2 * tensors]");
  TORCH_CHECK(ratios.scalar_type() == torch::kFloat32 && ratios.numel() == n_tensors, what, ": ratios: fp32 [tensors]");
  b2::LwArgs a;
  std::memset(&a, 0, sizeof(a));
  a.p = p.data_ptr<float>(); a.g = g.data_ptr<float>();
  a.m = states[0]->data_ptr<float>(); a.v = states.size() > 1 ? states[1]->data_ptr<float>() : nullptr;
  a.n = (size_t)p.numel();
  a.table = reinterpret_cast<const long long*>(table.data_ptr<int64_t>());
  a.n_chunks = (int)n_chunks; a.n_tensors = (int)n_tensors;
  a.partials = partials.data_ptr<float>(); a.tickets = reinterpret_cast<unsigned int*>(tickets.data_ptr<int32_t>());
  a.sums = sums.data_ptr<double>(); a.ratios = ratios.data_ptr<float>();
  a.zero_grad = zero_grad ? 1 : 0;
  const Clip c = clip_args(max_grad_norm, sqnorms, grad_norm_out, what);
  a.max_norm = c.max_norm; a.sqnorms = c.sq; a.n_buckets = c.n_buckets; a.grad_norm_out = c.gn;
  a.grad_scale = amp_scalar_ptr(grad_scale, p, what, "grad_scale");
  return a;
}

// The checked arguments of a sharded layer-wise launch (csrc/sharded_layerwise.cu): the per-rank pointer lists
// (sharded_peers), and this rank's table (sharded_layerwise_table), workspaces and state flats (`states`: m, then v (lamb) or
// LARS's gradient workspace), the state flats of at least one slice (n_vec / world x 4, x 8 with bf16) each.
std::pair<b2::LwArgs, Peers> sharded_layerwise_args(const char* what, bool lamb, bool bf16,
                                                    const std::vector<unsigned long long>& grads,
                                                    const std::vector<unsigned long long>& params,
                                                    const std::vector<unsigned long long>& sums,
                                                    const std::vector<unsigned long long>& sigs,
                                                    const std::vector<torch::Tensor*>& states, const ShardedLwTable& tab,
                                                    torch::Tensor& partials, torch::Tensor& tickets, torch::Tensor& ratios,
                                                    size_t n_vec, bool zero_grad, int rank, int world) {
  const Peers peers = sharded_peers(what, grads, params, &sums, sigs, n_vec, bf16, rank, world);
  const int64_t n_elems = (int64_t)n_vec * (bf16 ? 8 : 4);
  TORCH_CHECK(tab.rank == rank && tab.world == world && tab.n == n_elems, what, ": the table was built for rank ", tab.rank,
              " of ", tab.world, " on a bucket of ", tab.n, " elements; this launch is rank ", rank, " of ", world, " on ", n_elems);
  const torch::Tensor& table = tab.table;
  const int64_t n_chunks = tab.n_chunks;
  const int64_t shard = peers.shard;
  torch::Tensor& like = *states[0];
  check_flats({states.begin(), states.end()}, shard, true, "state shards (this rank's slice)", what);
  for (const torch::Tensor* t : {&table, (const torch::Tensor*)&partials, (const torch::Tensor*)&tickets,
                                 (const torch::Tensor*)&ratios}) {
    check_cuda_contig(*t, what);
    TORCH_CHECK(t->device() == like.device(), what, ": the table and the workspaces live on the state's device");
  }
  const int64_t n_tensors = tickets.numel();
  TORCH_CHECK(n_chunks >= 0 && n_chunks <= shard && n_tensors >= 1 && table.scalar_type() == torch::kInt64 &&
              table.numel() == (n_chunks + n_tensors) * b2::kLwRow, what, ": table: int64 of (chunks + tensors) * ", b2::kLwRow,
              " entries from sharded_layerwise_table, tickets: one per tensor");
  TORCH_CHECK(tickets.scalar_type() == torch::kInt32, what, ": tickets: int32 [tensors], zero before the first call");
  TORCH_CHECK(partials.scalar_type() == torch::kFloat32 && partials.numel() == 2 * n_chunks &&
              (n_chunks == 0 || (uintptr_t)partials.data_ptr() % 8 == 0), what, ": partials: fp32 [2 * chunks]");
  TORCH_CHECK(ratios.scalar_type() == torch::kFloat32 && ratios.numel() == n_tensors, what, ": ratios: fp32 [tensors]");
  b2::LwArgs a;
  std::memset(&a, 0, sizeof(a));
  a.m = states[0]->data_ptr<float>();
  (lamb ? a.v : a.g) = states[1]->data_ptr<float>();
  a.table = reinterpret_cast<const long long*>(table.data_ptr<int64_t>());
  a.n_chunks = (int)n_chunks; a.n_tensors = (int)n_tensors;
  a.partials = n_chunks > 0 ? partials.data_ptr<float>() : nullptr;
  a.tickets = reinterpret_cast<unsigned int*>(tickets.data_ptr<int32_t>());
  a.ratios = ratios.data_ptr<float>();
  a.zero_grad = zero_grad ? 1 : 0;
  return {a, peers};
}

// FlatAdafactor (csrc/adafactor.cu): the chunk table of one bucket (adafactor.h) from its tensors' offsets, shapes, strides,
// state offsets and groups, checked on the host and uploaded to `device`; returns (table, chunks, row / column partials,
// row_var means).  A tensor of dim > 1 is factored over its last two dimensions; its leading dimensions are merged where
// their strides allow and may number at most kAfMaxLead after that.
py::tuple adafactor_table(const std::vector<int64_t>& offsets, const std::vector<std::vector<int64_t>>& shapes,
                          const std::vector<std::vector<int64_t>>& strides, const std::vector<int64_t>& state_offsets,
                          const std::vector<int64_t>& groups, int64_t n, int64_t n_state, int64_t n_groups, torch::Device device) {
  const size_t nt = offsets.size();
  TORCH_CHECK(nt >= 1 && shapes.size() == nt && strides.size() == nt && state_offsets.size() == nt && groups.size() == nt,
              "adafactor_table: one offset, shape, strides, state offset and group per tensor, at least one tensor");
  TORCH_CHECK(nt < (size_t)INT32_MAX && n_groups >= 1 && n_groups <= b2::kMaxGroups, "adafactor_table: too many tensors, or a "
              "group count outside 1..", b2::kMaxGroups);
  const int64_t K = b2::kAfChunk;
  std::vector<int64_t> chunks, tens;
  int64_t end = 0, st_end = 0, rc = 0, means = 0;
  for (size_t t = 0; t < nt; ++t) {
    const auto& sh = shapes[t];
    const auto& sd = strides[t];
    TORCH_CHECK(sh.size() == sd.size(), "adafactor_table: tensor ", t, ": one stride per dimension");
    int64_t numel = 1, span = 0;
    for (size_t k = 0; k < sh.size(); ++k) {
      TORCH_CHECK(sh[k] >= 0 && sd[k] >= 0, "adafactor_table: tensor ", t, ": sizes and strides must be >= 0");
      numel *= sh[k];
      span += sh[k] > 0 ? (sh[k] - 1) * sd[k] : 0;
    }
    const int64_t o = offsets[t];
    TORCH_CHECK(numel < INT32_MAX && o >= end && o + numel <= n && (numel == 0 || span == numel - 1), "adafactor_table: tensor ", t,
                " at [", o, ", ", o + numel, ") must lie after the previous tensor inside the flat of ", n,
                " elements, be dense, and hold fewer than 2^31 elements");
    end = o + numel;
    const bool fac = sh.size() > 1;
    int64_t B = 1, R = 1, C = numel, sR = 0, sC = 1;
    std::vector<int64_t> lsz, lst;                         // merged leading dimensions, innermost first
    if (fac) {
      R = sh[sh.size() - 2]; C = sh.back(); sR = sd[sd.size() - 2]; sC = sd.back();
      for (size_t k = sh.size() - 2; k-- > 0;) {
        B *= sh[k];
        if (sh[k] == 1) continue;
        if (!lsz.empty() && sd[k] == lst.back() * lsz.back()) lsz.back() *= sh[k];
        else { lsz.push_back(sh[k]); lst.push_back(sd[k]); }
      }
      TORCH_CHECK(lsz.size() <= (size_t)b2::kAfMaxLead, "adafactor_table: tensor ", t, " has ", lsz.size(), " leading dimensions "
                  "after merging; at most ", b2::kAfMaxLead);
    } else {
      TORCH_CHECK(numel <= 1 || sd[0] == 1, "adafactor_table: tensor ", t, ": a 1-D tensor must be contiguous");
    }
    TORCH_CHECK(state_offsets[t] == st_end, "adafactor_table: tensor ", t, ": state at ", state_offsets[t], ", expected ", st_end,
                " (row_var, col_var or variance of each tensor in turn)");
    st_end += fac ? B * R + B * C : numel;
    TORCH_CHECK(groups[t] >= 0 && groups[t] < n_groups, "adafactor_table: tensor ", t, ": group ", groups[t], " outside [0, ",
                n_groups, ")");
    const int64_t first = (int64_t)chunks.size() / b2::kAfChunkRow;
    const bool whole = fac && R * C <= K;
    int64_t TR = 0, TC = 0, my_rc = rc;
    auto add = [&](int64_t b0, int64_t nb, int64_t r0, int64_t nr, int64_t c0, int64_t nc) {
      for (int64_t v : {(int64_t)t, b0, nb, r0, nr, c0, nc, (int64_t)0}) chunks.push_back(v);
    };
    if (numel > 0) {
      if (!fac) {
        for (int64_t c0 = 0; c0 < C; c0 += K) add(0, 1, 0, 1, c0, std::min(K, C - c0));
      } else if (whole) {
        const int64_t per = K / (R * C);
        for (int64_t b0 = 0; b0 < B; b0 += per) add(b0, std::min(per, B - b0), 0, R, 0, C);
      } else {
        TC = std::min<int64_t>(C, b2::kAfTileCols);
        TR = std::min<int64_t>(R, K / TC);
        TC = std::min<int64_t>(C, K / TR);
        for (int64_t b = 0; b < B; ++b)
          for (int64_t r0 = 0; r0 < R; r0 += TR)
            for (int64_t c0 = 0; c0 < C; c0 += TC) add(b, 1, r0, std::min(TR, R - r0), c0, std::min(TC, C - c0));
        rc += B * R * ((C + TC - 1) / TC) + B * C * ((R + TR - 1) / TR);
      }
    }
    const int64_t count = (int64_t)chunks.size() / b2::kAfChunkRow - first;
    int64_t row[b2::kAfTensorRow] = {0};
    row[b2::AF_OFFSET] = o; row[b2::AF_STATE] = state_offsets[t];
    row[b2::AF_B] = B; row[b2::AF_R] = R; row[b2::AF_C] = C; row[b2::AF_SR] = sR; row[b2::AF_SC] = sC;
    row[b2::AF_FIRST] = first; row[b2::AF_COUNT] = count; row[b2::AF_FACTORED] = fac ? 1 : 0; row[b2::AF_GROUP] = groups[t];
    row[b2::AF_WHOLE] = whole ? 1 : 0; row[b2::AF_TR] = TR; row[b2::AF_TC] = TC; row[b2::AF_RC] = my_rc;
    row[b2::AF_MEAN] = means; row[b2::AF_NLEAD] = (int64_t)lsz.size();
    for (size_t k = 0; k < lsz.size(); ++k) {            // stored outermost first
      row[b2::AF_LSIZE + k] = lsz[lsz.size() - 1 - k];
      row[b2::AF_LSTRIDE + k] = lst[lst.size() - 1 - k];
    }
    if (fac) means += B;
    tens.insert(tens.end(), row, row + b2::kAfTensorRow);
  }
  TORCH_CHECK(st_end <= n_state, "adafactor_table: the states need ", st_end, " elements, the state flat has ", n_state);
  const int64_t n_chunks = (int64_t)chunks.size() / b2::kAfChunkRow;
  TORCH_CHECK(n_chunks >= 1 && n_chunks < INT32_MAX, "adafactor_table: the tensors hold no element, or too many chunks");
  chunks.insert(chunks.end(), tens.begin(), tens.end());
  auto host = torch::tensor(chunks, torch::dtype(torch::kInt64));
  return py::make_tuple(host.to(device), n_chunks, rc, means);
}

b2::LrSchedule to_sched(const py::object& o) {
  b2::LrSchedule s;
  std::memset(&s, 0, sizeof(s));
  if (o.is_none()) return s;
  auto t = o.cast<py::tuple>();
  TORCH_CHECK(t.size() == 7, "lr_schedule: (kind, warmup, total, start, gamma, min_factor, milestones)");
  s.kind = t[0].cast<int>();
  TORCH_CHECK(s.kind >= b2::LRS_NONE && s.kind <= b2::LRS_COSINE, "lr_schedule: unknown kind ", s.kind);
  s.warmup = t[1].cast<long long>(); s.total = t[2].cast<long long>();
  s.start = t[3].cast<double>(); s.gamma = t[4].cast<double>(); s.min_factor = t[5].cast<double>();
  auto ms = t[6].cast<std::vector<long long>>();
  TORCH_CHECK((int)ms.size() <= b2::LRS_MAX_MILESTONES, "lr_schedule: at most 8 milestones");
  TORCH_CHECK(s.warmup >= 0 && (s.kind != b2::LRS_COSINE || s.total > s.warmup), "lr_schedule: bad warmup / total");
  s.n_milestones = (int)ms.size();
  for (size_t i = 0; i < ms.size(); ++i) s.milestones[i] = ms[i];
  return s;
}

// A capturable optimizer's device state (csrc/flat_scalars.h): the step counter (int64 CUDA [1], read as uint64), the table
// and the scalar block (uint8 CUDA, 16-byte aligned, at least flat_scalars_layout()'s bytes, on one device).
struct FlatState {
  b2::FlatHyper* table;
  unsigned long long* counter;
  b2::FlatScalars* block;
};
FlatState flat_state(const torch::Tensor& table, const torch::Tensor& counter, const torch::Tensor& block, const char* what) {
  TORCH_CHECK(counter.is_cuda() && counter.scalar_type() == torch::kInt64 && counter.numel() == 1, what,
              ": counter: int64 CUDA [1]");
  for (const torch::Tensor* t : {&table, &block})
    TORCH_CHECK(t->is_cuda() && t->is_contiguous() && t->scalar_type() == torch::kUInt8 && t->device() == counter.device() &&
                (uintptr_t)t->data_ptr() % 16 == 0, what, ": table / block: 16-byte aligned uint8 CUDA on the counter's device");
  TORCH_CHECK((size_t)table.numel() >= sizeof(b2::FlatHyper) && (size_t)block.numel() >= sizeof(b2::FlatScalars), what,
              ": table / block: at least ", sizeof(b2::FlatHyper), " / ", sizeof(b2::FlatScalars), " bytes");
  return {reinterpret_cast<b2::FlatHyper*>(table.data_ptr()), reinterpret_cast<unsigned long long*>(counter.data_ptr()),
          reinterpret_cast<b2::FlatScalars*>(block.data_ptr())};
}
// The block argument of a capturable update launch (see flat_state)
const b2::FlatScalars* flat_block(const torch::Tensor& block, const torch::Tensor& like, const char* what) {
  TORCH_CHECK(block.is_cuda() && block.is_contiguous() && block.scalar_type() == torch::kUInt8 && block.device() == like.device() &&
              (size_t)block.numel() >= sizeof(b2::FlatScalars) && (uintptr_t)block.data_ptr() % 16 == 0, what,
              ": block: 16-byte aligned uint8 CUDA of at least ", sizeof(b2::FlatScalars), " bytes on the parameters' device");
  return reinterpret_cast<const b2::FlatScalars*>(block.data_ptr());
}
// An optional group map of `n_ids` ids (null without groups)
const uint8_t* flat_map(const c10::optional<torch::Tensor>& map, int64_t n_ids, const char* what) {
  if (!map.has_value()) return nullptr;
  TORCH_CHECK(map->is_cuda() && map->is_contiguous() && map->scalar_type() == torch::kUInt8 && map->numel() >= n_ids, what,
              ": group_map: contiguous uint8 CUDA of at least ", n_ids, " ids (one per fp32 parameter vector)");
  return map->data_ptr<uint8_t>();
}

torch::Tensor tensor_from_ptr(unsigned long long ptr, int64_t numel, py::object dtype, int device) {
  auto st = torch::python::detail::py_object_to_dtype(dtype);
  auto opts = torch::TensorOptions().dtype(st).device(torch::kCUDA, device);
  return torch::from_blob((void*)(uintptr_t)ptr, {numel}, [](void*) {}, opts);
}

struct LoaderPy {
  std::unique_ptr<b2::NativeLoader> impl;
  torch::Tensor images, labels;   // keep the dataset alive
  std::vector<torch::Tensor> xs, ys;
  LoaderPy(torch::Tensor images_, torch::Tensor labels_, torch::Tensor index, int64_t batch, int n_buffers,
           bool shuffle, bool drop_last, bool raw_u8, double mean, double std, uint64_t seed, bool pin)
      : images(images_.contiguous()), labels(labels_.contiguous()) {
    TORCH_CHECK(!images.is_cuda() && images.scalar_type() == torch::kUInt8, "images: CPU uint8 tensor");
    TORCH_CHECK(!labels.is_cuda() && labels.scalar_type() == torch::kInt64, "labels: CPU int64 tensor");
    auto idx = index.to(torch::kInt64).contiguous();
    std::vector<int64_t> iv(idx.data_ptr<int64_t>(), idx.data_ptr<int64_t>() + idx.numel());
    const int64_t n = images.size(0);
    const int64_t item = images.numel() / std::max<int64_t>(n, 1);
    for (auto v : iv) TORCH_CHECK(v >= 0 && v < n, "index out of range");
    impl = std::make_unique<b2::NativeLoader>(images.data_ptr<uint8_t>(), labels.data_ptr<int64_t>(), item, std::move(iv),
                                              batch, n_buffers, shuffle, drop_last, raw_u8, (float)mean, (float)std,
                                              seed, pin);
    std::vector<int64_t> shape{batch, 1};
    for (int d = 1; d < images.dim(); ++d) shape.push_back(images.size(d));
    for (int i = 0; i < std::max(2, n_buffers); ++i) {
      auto& s = impl->slot(i);
      xs.push_back(torch::from_blob(s.x, shape, torch::TensorOptions().dtype(raw_u8 ? torch::kUInt8 : torch::kFloat32)));
      ys.push_back(torch::from_blob(s.y, {batch}, torch::TensorOptions().dtype(torch::kInt64)));
    }
  }
  py::object next() {
    int64_t count = 0;
    int slot;
    {
      py::gil_scoped_release nogil;
      slot = impl->next(&count);
    }
    if (slot < 0) return py::none();
    return py::make_tuple(xs[slot].narrow(0, 0, count), ys[slot].narrow(0, 0, count));
  }
};

struct ExecutorPy {
  std::unique_ptr<b2::StepExecutor> impl;
  LoaderPy* loader;
  std::vector<torch::Tensor> keep;
  ExecutorPy(LoaderPy& l, torch::Tensor params, torch::Tensor momentum, torch::Tensor grads,
             std::vector<unsigned long long> grad_ptrs, std::vector<unsigned long long> sig_ptrs, torch::Tensor step,
             torch::Tensor done_counter, torch::Tensor loss_acc, torch::Tensor in_dev, bool raw_u8, bool training, int rank,
             int world, uint64_t seed, int64_t sample_base, int64_t grad_stride, double lr, double mu, double p_drop,
             int max_in_flight, int cluster, torch::Tensor aux, std::vector<unsigned long long> inbox,
             torch::Tensor loss_hist, bool wire_bf16, c10::optional<torch::Tensor> grad_slots, c10::optional<torch::Tensor> factors,
             py::object lr_schedule, double weight_decay, bool nesterov, py::object max_grad_norm,
             c10::optional<torch::Tensor> clip_workspace, c10::optional<torch::Tensor> grad_norm_out)
      : loader(&l), keep{params, momentum, grads, step, done_counter, loss_acc, in_dev, aux, loss_hist} {
    TORCH_CHECK(l.impl->pinned(), "the native executor needs a pinned loader");
    TORCH_CHECK(raw_u8 == l.impl->raw(), "loader / trainer input dtype mismatch");
    const size_t block = (l.impl->block_bytes() + 255) / 256 * 256;
    const size_t nblk = (size_t)l.impl->num_slots();      // one device block and one loss snapshot per loader slot
    TORCH_CHECK(in_dev.is_cuda() && in_dev.scalar_type() == torch::kUInt8 && (size_t)in_dev.numel() >= nblk * block,
                "in_dev: CUDA uint8 buffer of >= num_slots * block bytes");
    TORCH_CHECK(loss_hist.is_cuda() && loss_hist.scalar_type() == torch::kFloat32 && (size_t)loss_hist.numel() >= 2 * nblk,
                "loss_hist: CUDA fp32 [num_slots, 2]");
    b2::StepConfig c;
    std::memset(&c, 0, sizeof(c));
    c.params = params.data_ptr<float>(); c.momentum = momentum.data_ptr<float>(); c.grads_local = grads.data_ptr<float>();
    for (size_t i = 0; i < grad_ptrs.size() && i < 8; ++i) c.grad_ptrs[i] = (void*)(uintptr_t)grad_ptrs[i];
    for (size_t i = 0; i < sig_ptrs.size() && i < 8; ++i) c.sig_ptrs[i] = (uint32_t*)(uintptr_t)sig_ptrs[i];
    c.step_counter = reinterpret_cast<unsigned long long*>(step.data_ptr());
    c.done_counter = reinterpret_cast<unsigned int*>(done_counter.data_ptr());
    c.loss_acc = loss_acc.data_ptr<float>();
    c.in_dev = in_dev.data_ptr<uint8_t>();
    c.in_stride = block;
    c.loss_hist = loss_hist.data_ptr<float>();
    c.B = (int)l.impl->batch(); c.x_u8 = raw_u8; c.training = training;
    c.rank = rank; c.world = world; c.seed = seed; c.sample_base = sample_base; c.grad_stride = grad_stride;
    c.lr = (float)lr; c.mu = (float)mu; c.p_drop = (float)p_drop; c.cluster = cluster;
    TORCH_CHECK(aux.is_cuda() && aux.scalar_type() == torch::kFloat32 && aux.numel() >= 13000, "aux: CUDA fp32 [13000]");
    c.aux = aux.data_ptr<float>();
    TORCH_CHECK(inbox.empty() || (int)inbox.size() == world, "inbox: one pointer per rank (or none)");
    for (size_t i = 0; i < inbox.size() && i < 8; ++i) c.inbox_ptrs[i] = (void*)(uintptr_t)inbox[i];
    c.push = !inbox.empty();
    if (grad_slots.has_value()) {    // one GPU, one CTA per sample: slots + factors reduced by reduce_sgd (no bucket)
      TORCH_CHECK(factors.has_value() && world == 1 && cluster <= 1, "grad_slots: one GPU, cluster 1");
      TORCH_CHECK(grad_slots->is_cuda() && grad_slots->scalar_type() == torch::kFloat32 && grad_slots->numel() >= c.B * (int64_t)21888 &&
                  factors->is_cuda() && factors->scalar_type() == torch::kFloat32 && factors->numel() >= c.B * (int64_t)384,
                  "grad_slots: [B, 21888] fp32, factors: [B, 384] fp32");
      keep.push_back(*grad_slots);
      keep.push_back(*factors);
      c.grad_slots = grad_slots->data_ptr<float>();
      c.factors = factors->data_ptr<float>();
    }
    c.wire_bf16 = wire_bf16 ? 1 : 0;
    c.sched = to_sched(lr_schedule);
    check_sgd_options(weight_decay, nesterov, mu, "StepExecutor");
    c.wd = (float)weight_decay; c.nesterov = nesterov ? 1 : 0;
    c.max_norm = check_max_grad_norm(max_grad_norm, "StepExecutor");
    c.clip_ws = clip_ws_ptr(c.max_norm, clip_workspace, params.numel(), "StepExecutor");
    c.grad_norm = grad_norm_ptr(grad_norm_out, "StepExecutor");
    if (c.clip_ws != nullptr) keep.push_back(*clip_workspace);
    if (c.grad_norm != nullptr) keep.push_back(*grad_norm_out);
    const int cap = std::max(1, l.impl->num_slots() - 2);
    c10::cuda::CUDAGuard guard(params.device());
    c10::cuda::getCurrentCUDAStream().synchronize();     // the executor's streams do not wait for work queued on this one
    impl = std::make_unique<b2::StepExecutor>(c, l.impl.get(), std::min(max_in_flight, cap));
  }
  py::tuple run(int64_t max_steps) {
    int pending = -1, epoch_done = 0;
    int64_t count = 0, done;
    {
      py::gil_scoped_release nogil;
      done = impl->run(max_steps, &pending, &count, &epoch_done);
    }
    if (done < 0) throw std::runtime_error("StepExecutor: " + impl->error());
    py::object tail = py::none();
    if (pending >= 0) tail = py::make_tuple(loader->xs[pending].narrow(0, 0, count), loader->ys[pending].narrow(0, 0, count));
    return py::make_tuple(done, tail, epoch_done != 0);
  }
};

// ---- SyncBatchNorm (csrc/batchnorm.cu)
int bn_dtype(const torch::Tensor& t, const char* what) {
  switch (t.scalar_type()) {
    case torch::kFloat32: return 0;
    case torch::kBFloat16: return 1;
    case torch::kHalf: return 2;
    default: TORCH_CHECK(false, "sync_batch_norm: ", what, " must be fp32, bf16 or fp16, got ", t.scalar_type());
  }
  return 0;
}

// One SyncBatchNorm kernel.  kind 0: statistics of x into ex; 1: y from ex (+ stats, running stats); 2: backward sums of
// dy, x into ex (+ grad_weight / grad_bias); 3: dx from ex and stats.  x is [N, C, ...], plain contiguous or channels-last
// (dy, y and dx share its strides); an [N, C] input (or any input with one element per (n, c)) is channels-last.
void bn_launch(int kind, torch::Tensor x, c10::optional<torch::Tensor> dy, c10::optional<torch::Tensor> out, torch::Tensor ex,
               torch::Tensor stats, c10::optional<torch::Tensor> tickets, c10::optional<torch::Tensor> weight,
               c10::optional<torch::Tensor> bias, c10::optional<torch::Tensor> running_mean,
               c10::optional<torch::Tensor> running_var, c10::optional<torch::Tensor> num_batches_tracked,
               c10::optional<torch::Tensor> grad_weight, c10::optional<torch::Tensor> grad_bias, double momentum, double eps,
               int max_blocks) {
  TORCH_CHECK(kind >= 0 && kind <= 3, "bn_launch: kind 0..3");
  TORCH_CHECK(x.is_cuda() && x.dim() >= 2, "sync_batch_norm: x must be a CUDA tensor of rank >= 2");
  const int dt = bn_dtype(x, "the input");
  const int64_t N = x.size(0), C = x.size(1);
  TORCH_CHECK(C >= 1 && C < (1ll << 30), "sync_batch_norm: channel count out of range");
  int64_t L = 1;
  for (int d = 2; d < x.dim(); ++d) L *= x.size(d);
  bool cl = false;
  if (L == 1 && x.is_contiguous()) cl = true;
  else if (x.is_contiguous()) cl = false;
  else if ((x.dim() == 4 && x.is_contiguous(at::MemoryFormat::ChannelsLast)) ||
           (x.dim() == 5 && x.is_contiguous(at::MemoryFormat::ChannelsLast3d))) cl = true;
  else TORCH_CHECK(false, "sync_batch_norm: x must be contiguous, channels_last or channels_last_3d");
  const int64_t M = cl ? N * L : N;
  std::vector<const torch::Tensor*> same;          // tensors laid out as x
  if (dy.has_value()) same.push_back(&*dy);
  if (out.has_value()) same.push_back(&*out);
  for (auto* t : same) {
    bool ok = t->is_cuda() && t->device() == x.device() && t->scalar_type() == x.scalar_type() && t->sizes() == x.sizes();
    for (int d = 0; ok && d < x.dim(); ++d) ok = x.size(d) == 1 || t->stride(d) == x.stride(d);   // size-1 strides are free
    TORCH_CHECK(ok, "sync_batch_norm: dy / y / dx must have the input's dtype, shape and strides");
  }
  TORCH_CHECK((kind == 0 || kind == 2 || out.has_value()) && (kind < 2 || dy.has_value()), "bn_launch: missing tensor");
  const int64_t es = x.element_size(), vw = 16 / es;
  bool vec = cl ? (C % vw == 0) : (L % vw == 0);
  vec = vec && (uintptr_t)x.data_ptr() % 16 == 0;
  for (auto* t : same) vec = vec && (uintptr_t)t->data_ptr() % 16 == 0;
  const int64_t n_ex = kind < 2 ? 1 + 2 * C : 2 * C;
  TORCH_CHECK(ex.is_cuda() && ex.is_contiguous() && ex.scalar_type() == torch::kFloat64 && ex.numel() >= n_ex,
              "sync_batch_norm: the exchange buffer must be contiguous fp64 CUDA of at least ", n_ex, " elements");
  TORCH_CHECK(stats.is_cuda() && stats.is_contiguous() && stats.scalar_type() == torch::kFloat64 && stats.numel() >= 2 * C + 1,
              "sync_batch_norm: stats must be contiguous fp64 CUDA [2C + 1]");
  auto param = [&](const c10::optional<torch::Tensor>& t, const char* what, int* code) -> void* {
    if (!t.has_value()) return nullptr;
    TORCH_CHECK(t->is_cuda() && t->device() == x.device() && t->is_contiguous() && t->numel() == C, "sync_batch_norm: ", what,
                " must be a contiguous CUDA tensor of C elements");
    const int c = bn_dtype(*t, what);
    TORCH_CHECK(c == 0 || c == dt, "sync_batch_norm: ", what, " must be fp32 or the input's dtype");
    TORCH_CHECK(*code < 0 || *code == c, "sync_batch_norm: weight, bias and their gradients (and the running stats) share a dtype");
    *code = c;
    return t->data_ptr();
  };
  b2::bn::Args a{};
  int pw = -1, pr = -1;
  a.x = x.data_ptr();
  if (kind == 1) a.y = out->data_ptr();
  if (kind == 3) a.dx = out->data_ptr();
  if (kind >= 2) a.dy = dy->data_ptr();
  a.w = param(weight, "weight", &pw);
  a.b = param(bias, "bias", &pw);
  a.gw = param(grad_weight, "grad_weight", &pw);
  a.gb = param(grad_bias, "grad_bias", &pw);
  a.rmean = param(running_mean, "running_mean", &pr);
  a.rvar = param(running_var, "running_var", &pr);
  TORCH_CHECK((a.rmean == nullptr) == (a.rvar == nullptr), "sync_batch_norm: running_mean and running_var go together");
  a.pw = pw < 0 ? 0 : pw;
  a.pr = pr < 0 ? 0 : pr;
  if (num_batches_tracked.has_value()) {
    TORCH_CHECK(num_batches_tracked->is_cuda() && num_batches_tracked->scalar_type() == torch::kInt64 &&
                num_batches_tracked->numel() == 1, "sync_batch_norm: num_batches_tracked must be a CUDA int64 scalar");
    a.nbt = reinterpret_cast<const long long*>(num_batches_tracked->data_ptr());
  }
  a.momentum = momentum;
  a.eps = eps;
  a.ex = ex.data_ptr<double>();
  a.n_ex = (int)ex.numel();
  a.stats = stats.data_ptr<double>();
  a.count = (long long)(N * L);
  a.C = (int)C;
  c10::cuda::CUDAGuard guard(x.device());
  torch::Tensor part;
  if (kind == 0 || kind == 2) {
    TORCH_CHECK(tickets.has_value() && tickets->is_cuda() && tickets->is_contiguous() && tickets->scalar_type() == torch::kInt32 &&
                tickets->numel() >= C, "sync_batch_norm: tickets must be a contiguous int32 CUDA tensor of at least C elements, "
                "zero before its first use");
    unsigned int g[2];
    ck_cuda(b2_bn_launch(kind, dt, vec, cl, M, L, max_blocks, &a, g, cur_stream()), "bn geometry");
    part = torch::empty({(int64_t)g[1] * 2 * C}, x.options().dtype(torch::kFloat64));
    a.part = part.data_ptr<double>();
    a.tickets = reinterpret_cast<unsigned int*>(tickets->data_ptr());
  }
  ck_cuda(b2_bn_launch(kind, dt, vec, cl, M, L, max_blocks, &a, nullptr, cur_stream()), "sync_batch_norm launch");
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "dist_tuto.pth_b200 native runtime: symmetric memory, fused sm_90a kernels, native loader";

  // ------------------------------------------------------------------ symmetric memory
  m.def("symm_caps", [](int dev) { int c[3]; ck_symm(b2_symm_caps(dev, c), "symm_caps"); return std::vector<int>{c[0], c[1], c[2]}; });
  m.def("symm_granularity", [](int dev, int ndev, bool mc) { size_t g = 0; ck_symm(b2_symm_granularity(dev, ndev, mc, &g), "granularity"); return g; });
  m.def("symm_create", [](int dev, size_t bytes) { unsigned long long h; int fd; ck_symm(b2_symm_create(dev, bytes, &h, &fd), "symm_create"); return py::make_tuple(h, fd); });
  m.def("symm_import", [](int fd) { unsigned long long h; ck_symm(b2_symm_import(fd, &h), "symm_import"); return h; });
  m.def("symm_map", [](int dev, unsigned long long h, size_t bytes, size_t align) { unsigned long long p; ck_symm(b2_symm_map(dev, h, bytes, align, &p), "symm_map"); return p; });
  m.def("symm_unmap", [](unsigned long long p, size_t bytes) { ck_symm(b2_symm_unmap(p, bytes), "symm_unmap"); });
  m.def("symm_release", [](unsigned long long h) { ck_symm(b2_symm_release(h), "symm_release"); });
  m.def("mc_create", [](int ndev, size_t bytes) { unsigned long long h; int fd; ck_symm(b2_mc_create(ndev, bytes, &h, &fd), "mc_create"); return py::make_tuple(h, fd); });
  m.def("mc_add_device", [](unsigned long long mc, int dev) { ck_symm(b2_mc_add_device(mc, dev), "mc_add_device"); });
  m.def("mc_bind", [](unsigned long long mc, unsigned long long mem, size_t bytes) { ck_symm(b2_mc_bind(mc, mem, bytes), "mc_bind"); });
  m.def("mc_unbind", [](unsigned long long mc, int dev, size_t bytes) { ck_symm(b2_mc_unbind(mc, dev, bytes), "mc_unbind"); });
  m.def("ipc_alloc", [](size_t bytes) {
    unsigned long long p; unsigned char h[64];
    ck_symm(b2_ipc_alloc(bytes, &p, h), "ipc_alloc");
    return py::make_tuple(p, py::bytes(reinterpret_cast<const char*>(h), 64));
  });
  m.def("ipc_open", [](py::bytes handle) {
    std::string s = handle;
    TORCH_CHECK(s.size() == 64, "ipc handle must be 64 bytes");
    unsigned long long p; ck_symm(b2_ipc_open(reinterpret_cast<const unsigned char*>(s.data()), &p), "ipc_open");
    return p;
  });
  m.def("ipc_close", [](unsigned long long p) { b2_ipc_close(p); });
  m.def("ipc_free", [](unsigned long long p) { b2_ipc_free(p); });
  m.def("tensor_from_ptr", &tensor_from_ptr, "wrap device memory as a 1-D tensor (no ownership)");

  // ------------------------------------------------------------------ collectives
  // op: 0 SUM, 1 PRODUCT, 2 MAX, 3 MIN (reductions; root >= 0 stores on that rank only), 4 broadcast from root, 5 all-gather
  // (n_vec counts the output, world x the per-rank input; root >= 0: gather to that rank), 6 scatter from root (n_vec counts
  // the root's input, world x the per-rank output).  The raw moves take any dtype and copy bytes.
  // dtype (reductions): the kernels' wire dtype code, 0 fp32, 1 bf16, 2 fp16, 3 fp64, 4 int8, 5 uint8, 6 int32, 7 int64,
  // 8 bool; -1 takes fp32 or bf16 from `bf16`.  Codes 2..8 take locals of that dtype only, no scale, no bf16 wire and no NVLS.
  static const torch::ScalarType kDtypes[] = {torch::kFloat32, torch::kBFloat16, torch::kFloat16, torch::kFloat64, torch::kInt8,
                                              torch::kUInt8, torch::kInt32, torch::kInt64, torch::kBool};
  auto collective = [](const char* what, int op, int variant, bool bf16, const std::vector<unsigned long long>& bufs,
                       const std::vector<unsigned long long>& sigs, unsigned long long mc, const c10::optional<torch::Tensor>& src,
                       const c10::optional<torch::Tensor>& dst, size_t n_vec, double scale, int root, int rank, int world,
                       int max_blocks, const std::vector<unsigned long long>& inbox, size_t ll_cap, int dtype = -1) {
    check_world(rank, world, what);
    TORCH_CHECK(variant >= 0 && variant <= 3, what, ": variant must be 0 (one-shot), 1 (two-shot), 2 (NVLS) or 3 (LL), got ",
                variant);
    TORCH_CHECK((int)bufs.size() == world && (int)sigs.size() == world, what, ": one buffer and one signal pad per rank, got ",
                bufs.size(), " and ", sigs.size(), " for world ", world);
    TORCH_CHECK(variant == 3 ? (int)inbox.size() == world : inbox.empty() || (int)inbox.size() == world,
                what, ": one LL inbox per rank, got ", inbox.size(), " for world ", world);
    const bool segmented = op == 5 || op == 6;              // all-gather, gather, scatter: one segment per rank
    TORCH_CHECK((variant != 1 && variant != 2 && !segmented) || n_vec % (size_t)world == 0,
                what, ": two-shot, NVLS, all-gather, gather and scatter split n_vec into world slices, so n_vec must be a "
                "multiple of world (pad the buffer), got n_vec ", n_vec, " for world ", world);
    TORCH_CHECK(root >= -1 && root < world, what, ": root must be -1 (every rank) or in [0, world), got ", root,
                " for world ", world);
    TORCH_CHECK(op == 0 || scale == 1.0, what, ": scale applies to SUM only, got ", scale, " for op ", op);
    TORCH_CHECK(variant != 2 || (op == 0 && root < 0), what, ": NVLS runs the SUM all-reduce only");
    TORCH_CHECK(variant != 3 || (segmented ? n_vec / world : n_vec) <= ll_cap, what, ": LL pushes ",
                segmented ? n_vec / world : n_vec, " vectors per rank, more than the inbox holds (", ll_cap, ")");
    TORCH_CHECK(dtype >= -1 && dtype <= 8, what, ": dtype must be -1 (fp32 / bf16 from the bf16 flag) or a code in 0..8, got ",
                dtype);
    TORCH_CHECK(dtype < 0 || dtype >= 2 || dtype == (int)bf16, what, ": dtype ", dtype, " contradicts the bf16 flag (",
                bf16, ")");
    const bool narrow = dtype >= 2;                        // a dtype beyond fp32 / bf16
    TORCH_CHECK(!narrow || !bf16, what, ": a bf16 wire is for fp32 / bf16 tensors, not dtype ", dtype);
    TORCH_CHECK(!narrow || scale == 1.0, what, ": scale applies to fp32 / bf16 SUM only, got ", scale, " for dtype ", dtype);
    TORCH_CHECK(!narrow || variant != 2, what, ": NVLS reduces fp32 / bf16 only, not dtype ", dtype);
    TORCH_CHECK(dtype != 8 || op != 0, what, ": a bool SUM is a MAX (as torch.distributed maps it); pass op 2");
    if (narrow) {
      for (const auto* t : {&src, &dst})
        TORCH_CHECK(!t->has_value() || (*t)->scalar_type() == kDtypes[dtype], what, ": ", t == &src ? "src" : "dst",
                    " is ", (*t)->scalar_type(), " but dtype ", dtype, " is ", kDtypes[dtype]);
    }
    PeerPtrs b = to_ptrs(bufs); SignalPadsH s = to_sig(sigs);
    PeerPtrs ib = to_ptrs(inbox);
    const void* sp = nullptr; void* dp = nullptr; int sf = 0, df = 0;
    if (src.has_value()) { check_cuda_contig(*src, "src"); sp = src->data_ptr(); sf = src->scalar_type() == torch::kFloat32 && bf16; }
    if (dst.has_value()) { check_cuda_contig(*dst, "dst"); dp = dst->data_ptr(); df = dst->scalar_type() == torch::kFloat32 && bf16; }
    TORCH_CHECK(op == 0 || (sf == 0 && df == 0), what, ": a bf16 wire for fp32 tensors is for SUM only");
    ck_cuda(b2_allreduce_dtype_launch(variant, dtype < 0 ? (int)bf16 : dtype, &b, &s, (void*)(uintptr_t)mc, sp, sf, dp, df,
                                      n_vec, (float)scale, rank, world, max_blocks, inbox.empty() ? nullptr : &ib, ll_cap, op,
                                      root, cur_stream()), what);
  };
  m.def("allreduce", [collective](int variant, bool bf16, std::vector<unsigned long long> bufs, std::vector<unsigned long long> sigs,
                                  unsigned long long mc, c10::optional<torch::Tensor> src, c10::optional<torch::Tensor> dst,
                                  size_t n_vec, double scale, int rank, int world, int max_blocks, std::vector<unsigned long long> inbox,
                                  size_t ll_cap, int op, int root, int dtype) {
    TORCH_CHECK(op >= 0 && op <= 3, "allreduce: op must be 0 (SUM), 1 (PRODUCT), 2 (MAX) or 3 (MIN), got ", op);
    collective("allreduce", op, variant, bf16, bufs, sigs, mc, src, dst, n_vec, scale, root, rank, world, max_blocks, inbox, ll_cap,
               dtype);
  }, py::arg("variant"), py::arg("bf16"), py::arg("bufs"), py::arg("sigs"), py::arg("mc"), py::arg("src"), py::arg("dst"),
     py::arg("n_vec"), py::arg("scale"), py::arg("rank"), py::arg("world"), py::arg("max_blocks") = 0,
     py::arg("inbox") = std::vector<unsigned long long>(), py::arg("ll_cap") = 0, py::arg("op") = 0, py::arg("root") = -1,
     py::arg("dtype") = -1);
  m.def("broadcast", [collective](int variant, std::vector<unsigned long long> bufs, std::vector<unsigned long long> sigs,
                                  c10::optional<torch::Tensor> src, c10::optional<torch::Tensor> dst, size_t n_vec, int root,
                                  int rank, int world, int max_blocks, std::vector<unsigned long long> inbox, size_t ll_cap) {
    TORCH_CHECK(root >= 0, "broadcast: root must be in [0, world), got ", root);
    collective("broadcast", 4, variant, false, bufs, sigs, 0, src, dst, n_vec, 1.0, root, rank, world, max_blocks, inbox, ll_cap);
  }, py::arg("variant"), py::arg("bufs"), py::arg("sigs"), py::arg("src"), py::arg("dst"), py::arg("n_vec"), py::arg("root"),
     py::arg("rank"), py::arg("world"), py::arg("max_blocks") = 0, py::arg("inbox") = std::vector<unsigned long long>(),
     py::arg("ll_cap") = 0);
  m.def("allgather", [collective](int variant, std::vector<unsigned long long> bufs, std::vector<unsigned long long> sigs,
                                  c10::optional<torch::Tensor> src, c10::optional<torch::Tensor> dst, size_t n_vec, int rank,
                                  int world, int max_blocks, std::vector<unsigned long long> inbox, size_t ll_cap) {
    collective("allgather", 5, variant, false, bufs, sigs, 0, src, dst, n_vec, 1.0, -1, rank, world, max_blocks, inbox, ll_cap);
  }, py::arg("variant"), py::arg("bufs"), py::arg("sigs"), py::arg("src"), py::arg("dst"), py::arg("n_vec"), py::arg("rank"),
     py::arg("world"), py::arg("max_blocks") = 0, py::arg("inbox") = std::vector<unsigned long long>(), py::arg("ll_cap") = 0);
  // gather / scatter: every rank of one call must pass the same src / dst nullness (the one-shot and two-shot barriers depend
  // on it); src of a scatter and dst of a gather are used on the root only.
  m.def("gather", [collective](int variant, std::vector<unsigned long long> bufs, std::vector<unsigned long long> sigs,
                               c10::optional<torch::Tensor> src, c10::optional<torch::Tensor> dst, size_t n_vec, int root,
                               int rank, int world, int max_blocks, std::vector<unsigned long long> inbox, size_t ll_cap) {
    TORCH_CHECK(root >= 0, "gather: root must be in [0, world), got ", root);
    collective("gather", 5, variant, false, bufs, sigs, 0, src, dst, n_vec, 1.0, root, rank, world, max_blocks, inbox, ll_cap);
  }, py::arg("variant"), py::arg("bufs"), py::arg("sigs"), py::arg("src"), py::arg("dst"), py::arg("n_vec"), py::arg("root"),
     py::arg("rank"), py::arg("world"), py::arg("max_blocks") = 0, py::arg("inbox") = std::vector<unsigned long long>(),
     py::arg("ll_cap") = 0);
  m.def("scatter", [collective](int variant, std::vector<unsigned long long> bufs, std::vector<unsigned long long> sigs,
                                c10::optional<torch::Tensor> src, c10::optional<torch::Tensor> dst, size_t n_vec, int root,
                                int rank, int world, int max_blocks, std::vector<unsigned long long> inbox, size_t ll_cap) {
    TORCH_CHECK(root >= 0, "scatter: root must be in [0, world), got ", root);
    collective("scatter", 6, variant, false, bufs, sigs, 0, src, dst, n_vec, 1.0, root, rank, world, max_blocks, inbox, ll_cap);
  }, py::arg("variant"), py::arg("bufs"), py::arg("sigs"), py::arg("src"), py::arg("dst"), py::arg("n_vec"), py::arg("root"),
     py::arg("rank"), py::arg("world"), py::arg("max_blocks") = 0, py::arg("inbox") = std::vector<unsigned long long>(),
     py::arg("ll_cap") = 0);
  // reduce-scatter / all-to-all: n_vec counts one rank's input, world segments of n_vec / world vectors.  variant 0 pull
  // (one-shot, two-shot and NVLS all map to it on the Python side), 3 LL.  src null: the input is this rank's buffer; dst
  // null (reduce-scatter only): the output is segment `rank` of it.  Every rank of one call must pass the same n_vec.
  auto segments = [](const char* what, int variant, const std::vector<unsigned long long>& bufs,
                     const std::vector<unsigned long long>& sigs, const c10::optional<torch::Tensor>& src,
                     const c10::optional<torch::Tensor>& dst, size_t n_vec, int rank, int world,
                     const std::vector<unsigned long long>& inbox, size_t ll_cap, PeerPtrs* b, SignalPadsH* s, PeerPtrs* ib) {
    check_world(rank, world, what);
    TORCH_CHECK(variant == 0 || variant == 3, what, ": variant must be 0 (pull) or 3 (LL), got ", variant);
    TORCH_CHECK((int)bufs.size() == world && (int)sigs.size() == world, what, ": one buffer and one signal pad per rank, got ",
                bufs.size(), " and ", sigs.size(), " for world ", world);
    TORCH_CHECK(variant == 3 ? (int)inbox.size() == world : inbox.empty() || (int)inbox.size() == world,
                what, ": one LL inbox per rank, got ", inbox.size(), " for world ", world);
    TORCH_CHECK(n_vec % (size_t)world == 0, what, ": n_vec holds world segments, so it must be a multiple of world, got n_vec ",
                n_vec, " for world ", world);
    TORCH_CHECK(variant != 3 || n_vec / world <= ll_cap, what, ": LL pushes ", n_vec / world,
                " vectors per peer, more than the inbox holds (", ll_cap, ")");
    for (const auto* t : {&src, &dst}) {
      if (t->has_value()) {
        check_cuda_contig(**t, t == &src ? "src" : "dst");
        TORCH_CHECK((size_t)(*t)->nbytes() >= n_vec * 16, what, ": ", t == &src ? "src" : "dst", " holds ", (*t)->nbytes(),
                    " bytes, the call needs ", n_vec * 16);
      }
    }
    *b = to_ptrs(bufs); *s = to_sig(sigs); *ib = to_ptrs(inbox);
  };
  m.def("reduce_scatter", [segments](int variant, std::vector<unsigned long long> bufs, std::vector<unsigned long long> sigs,
                                     c10::optional<torch::Tensor> src, c10::optional<torch::Tensor> dst, size_t n_vec, int rank,
                                     int world, int max_blocks, std::vector<unsigned long long> inbox, size_t ll_cap, int op,
                                     int dtype) {
    TORCH_CHECK(op >= 0 && op <= 3, "reduce_scatter: op must be 0 (SUM), 1 (PRODUCT), 2 (MAX) or 3 (MIN), got ", op);
    TORCH_CHECK(dtype >= 0 && dtype <= 8, "reduce_scatter: dtype must be a code in 0..8, got ", dtype);
    TORCH_CHECK(dtype != 8 || op != 0, "reduce_scatter: a bool SUM is a MAX (as torch.distributed maps it); pass op 2");
    for (const auto* t : {&src, &dst})
      TORCH_CHECK(!t->has_value() || (*t)->scalar_type() == kDtypes[dtype], "reduce_scatter: ", t == &src ? "src" : "dst",
                  " is ", (*t)->scalar_type(), " but dtype ", dtype, " is ", kDtypes[dtype]);
    PeerPtrs b, ib; SignalPadsH s;
    segments("reduce_scatter", variant, bufs, sigs, src, c10::nullopt, n_vec, rank, world, inbox, ll_cap, &b, &s, &ib);
    if (dst.has_value()) {
      check_cuda_contig(*dst, "dst");
      TORCH_CHECK((size_t)dst->nbytes() >= n_vec / world * 16, "reduce_scatter: dst holds ", dst->nbytes(),
                  " bytes, one segment is ", n_vec / world * 16);
    }
    ck_cuda(b2_reduce_scatter_launch(variant, dtype, op, &b, &s, src.has_value() ? src->data_ptr() : nullptr,
                                     dst.has_value() ? dst->data_ptr() : nullptr, n_vec, rank, world, max_blocks,
                                     inbox.empty() ? nullptr : &ib, ll_cap, cur_stream()), "reduce_scatter");
  }, py::arg("variant"), py::arg("bufs"), py::arg("sigs"), py::arg("src"), py::arg("dst"), py::arg("n_vec"), py::arg("rank"),
     py::arg("world"), py::arg("max_blocks") = 0, py::arg("inbox") = std::vector<unsigned long long>(), py::arg("ll_cap") = 0,
     py::arg("op") = 0, py::arg("dtype") = 0);
  m.def("alltoall", [segments](int variant, std::vector<unsigned long long> bufs, std::vector<unsigned long long> sigs,
                               c10::optional<torch::Tensor> src, torch::Tensor dst, size_t n_vec, int rank, int world,
                               int max_blocks, std::vector<unsigned long long> inbox, size_t ll_cap) {
    PeerPtrs b, ib; SignalPadsH s;
    segments("alltoall", variant, bufs, sigs, src, dst, n_vec, rank, world, inbox, ll_cap, &b, &s, &ib);
    ck_cuda(b2_alltoall_launch(variant, &b, &s, src.has_value() ? src->data_ptr() : nullptr, dst.data_ptr(), n_vec, rank, world,
                               max_blocks, inbox.empty() ? nullptr : &ib, ll_cap, cur_stream()), "alltoall");
  }, py::arg("variant"), py::arg("bufs"), py::arg("sigs"), py::arg("src"), py::arg("dst"), py::arg("n_vec"), py::arg("rank"),
     py::arg("world"), py::arg("max_blocks") = 0, py::arg("inbox") = std::vector<unsigned long long>(), py::arg("ll_cap") = 0);
  // all-to-allv: srcs[d] (its first src_bytes[d] bytes) goes to rank d; what rank p sends lands in dsts[p], at most
  // dst_bytes[p] bytes of it.  bufs: staging buffers of header + 2 x world x chunk bytes (alltoallv_config).  Any dtype and
  // alignment; every rank of one call must run it, whatever its lengths.
  m.def("alltoallv_config", [] {
    size_t chunk = 0, header = 0;
    b2_alltoallv_config(&chunk, &header);
    return py::make_tuple(chunk, header);
  }, "(bytes per pair and round, header bytes) of the all-to-allv staging buffer");
  m.def("alltoallv", [](std::vector<unsigned long long> bufs, std::vector<unsigned long long> sigs,
                        std::vector<torch::Tensor> srcs, std::vector<long long> src_bytes, std::vector<torch::Tensor> dsts,
                        std::vector<long long> dst_bytes, int rank, int world, int max_blocks) {
    check_world(rank, world, "alltoallv");
    TORCH_CHECK((int)bufs.size() == world && (int)sigs.size() == world, "alltoallv: one buffer and one signal pad per rank, got ",
                bufs.size(), " and ", sigs.size(), " for world ", world);
    TORCH_CHECK((int)srcs.size() == world && (int)src_bytes.size() == world && (int)dsts.size() == world &&
                (int)dst_bytes.size() == world, "alltoallv: one source, one destination and their byte counts per rank, got ",
                srcs.size(), ", ", src_bytes.size(), ", ", dsts.size(), " and ", dst_bytes.size(), " for world ", world);
    const void* sp[B2_MAX_RANKS];
    void* dp[B2_MAX_RANKS];
    unsigned long long sn[B2_MAX_RANKS], dn[B2_MAX_RANKS];
    for (int r = 0; r < world; ++r) {
      check_cuda_contig(srcs[r], "alltoallv: src");
      check_cuda_contig(dsts[r], "alltoallv: dst");
      TORCH_CHECK(src_bytes[r] >= 0 && (size_t)src_bytes[r] <= (size_t)srcs[r].nbytes(), "alltoallv: ", src_bytes[r],
                  " bytes for rank ", r, " from a source of ", srcs[r].nbytes());
      TORCH_CHECK(dst_bytes[r] >= 0 && (size_t)dst_bytes[r] <= (size_t)dsts[r].nbytes(), "alltoallv: ", dst_bytes[r],
                  " bytes from rank ", r, " into a destination of ", dsts[r].nbytes());
      sp[r] = srcs[r].data_ptr(); sn[r] = (unsigned long long)src_bytes[r];
      dp[r] = dsts[r].data_ptr(); dn[r] = (unsigned long long)dst_bytes[r];
    }
    PeerPtrs b = to_ptrs(bufs);
    SignalPadsH s = to_sig(sigs);
    ck_cuda(b2_alltoallv_launch(&b, &s, sp, sn, dp, dn, rank, world, max_blocks, cur_stream()), "alltoallv");
  }, py::arg("bufs"), py::arg("sigs"), py::arg("srcs"), py::arg("src_bytes"), py::arg("dsts"), py::arg("dst_bytes"),
     py::arg("rank"), py::arg("world"), py::arg("max_blocks") = 0);
  m.def("barrier", [](std::vector<unsigned long long> sigs, int rank, int world) {
    check_world(rank, world, "barrier");
    TORCH_CHECK((int)sigs.size() == world, "barrier: one signal pad per rank, got ", sigs.size(), " for world ", world);
    SignalPadsH s = to_sig(sigs);
    ck_cuda(b2_barrier_launch(&s, rank, world, cur_stream()), "barrier launch");
  });

  // ------------------------------------------------------------------ point-to-point (csrc/p2p.cu)
  // bufs / sigs: the mailbox data and signal pad of every rank.  Both sides of a transfer must pass the same byte count (as
  // with NCCL); a zero-byte message launches nothing.  Messages between one pair are matched in issue order.
  m.def("p2p_config", [] {
    int ctas = 0, slots = 0, pad_words = 0;
    size_t chunk = 0;
    b2_p2p_config(&ctas, &slots, &chunk, &pad_words);
    return py::make_tuple(ctas, slots, chunk, pad_words);
  }, "(CTAs per transfer, slots per CTA, bytes per slot, signal-pad words) of the point-to-point mailbox");
  // A stream of its own, not one of torch's pooled streams (handed out round robin, so two of them can be one CUDA stream):
  // a send and a receive that wait for their peers must never be queued on one stream.
  m.def("stream_create", [](int device) {
    c10::cuda::CUDAGuard guard(device);
    cudaStream_t s = nullptr;
    ck_cuda((int)cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking), "cudaStreamCreateWithFlags");
    return (unsigned long long)(uintptr_t)s;
  }, py::arg("device"));
  m.def("stream_destroy", [](unsigned long long s) {
    ck_cuda((int)cudaStreamDestroy((cudaStream_t)(uintptr_t)s), "cudaStreamDestroy");
  }, py::arg("stream"));
  auto p2p = [](const char* what, bool send, const std::vector<unsigned long long>& bufs,
                const std::vector<unsigned long long>& sigs, const torch::Tensor& t, int peer, int rank, int world) {
    check_world(rank, world, what);
    TORCH_CHECK(world >= 2, what, ": a point-to-point transfer needs a world of at least 2, got ", world);
    TORCH_CHECK(peer >= 0 && peer < world, what, ": peer ", peer, " is outside [0, ", world, ")");
    TORCH_CHECK(peer != rank, what, ": rank ", rank, " cannot be its own peer");
    TORCH_CHECK((int)bufs.size() == world && (int)sigs.size() == world, what, ": one mailbox and one signal pad per rank, got ",
                bufs.size(), " and ", sigs.size(), " for world ", world);
    check_cuda_contig(t, send ? "src" : "dst");
    TORCH_CHECK((uintptr_t)t.data_ptr() % 16 == 0, what, ": the tensor must be 16-byte aligned");
    const size_t nbytes = (size_t)t.numel() * t.element_size();
    if (nbytes == 0) return;
    PeerPtrs b = to_ptrs(bufs); SignalPadsH s = to_sig(sigs);
    c10::cuda::CUDAGuard guard(t.device());
    ck_cuda(send ? b2_p2p_send_launch(&b, &s, t.data_ptr(), nbytes, rank, peer, world, cur_stream())
                 : b2_p2p_recv_launch(&b, &s, t.data_ptr(), nbytes, rank, peer, world, cur_stream()), what);
  };
  m.def("p2p_send", [p2p](std::vector<unsigned long long> bufs, std::vector<unsigned long long> sigs, torch::Tensor src, int peer,
                          int rank, int world) { p2p("p2p_send", true, bufs, sigs, src, peer, rank, world); },
        py::arg("bufs"), py::arg("sigs"), py::arg("src"), py::arg("peer"), py::arg("rank"), py::arg("world"));
  m.def("p2p_recv", [p2p](std::vector<unsigned long long> bufs, std::vector<unsigned long long> sigs, torch::Tensor dst, int peer,
                          int rank, int world) { p2p("p2p_recv", false, bufs, sigs, dst, peer, rank, world); },
        py::arg("bufs"), py::arg("sigs"), py::arg("dst"), py::arg("peer"), py::arg("rank"), py::arg("world"));
  m.def("p2p_batch_capacity", [] { return b2_p2p_batch_capacity(); }, "the most ops one p2p_batch takes");
  // ops: [(send, tensor, peer)], all in one launch on the current stream (torch's batch_isend_irecv).  Each pair's messages
  // match in list order, against batches or single p2p_send / p2p_recv on the peer alike; zero-byte ops are dropped.
  m.def("p2p_batch", [](std::vector<unsigned long long> bufs, std::vector<unsigned long long> sigs,
                        std::vector<std::tuple<bool, torch::Tensor, int>> ops, int rank, int world) {
    const char* what = "p2p_batch";
    check_world(rank, world, what);
    TORCH_CHECK(world >= 2, what, ": a point-to-point transfer needs a world of at least 2, got ", world);
    TORCH_CHECK((int)bufs.size() == world && (int)sigs.size() == world, what, ": one mailbox and one signal pad per rank, got ",
                bufs.size(), " and ", sigs.size(), " for world ", world);
    TORCH_CHECK((long long)ops.size() <= b2_p2p_batch_capacity(), what, ": at most ", b2_p2p_batch_capacity(),
                " ops per batch, got ", ops.size());
    for (const auto& op : ops) {
      const int p = std::get<2>(op);
      TORCH_CHECK(p >= 0 && p < world, what, ": peer ", p, " is outside [0, ", world, ")");
      TORCH_CHECK(p != rank, what, ": rank ", rank, " cannot be its own peer");
    }
    std::vector<int> send, peer;
    std::vector<void*> msg;
    std::vector<size_t> nbytes;
    for (const auto& op : ops) {
      const torch::Tensor& t = std::get<1>(op);
      const int p = std::get<2>(op);
      check_cuda_contig(t, "every tensor");
      TORCH_CHECK(t.device() == std::get<1>(ops[0]).device(), what, ": every tensor must be on one device");
      TORCH_CHECK((uintptr_t)t.data_ptr() % 16 == 0, what, ": every tensor must be 16-byte aligned");
      const size_t n = (size_t)t.numel() * t.element_size();
      if (n == 0) continue;
      send.push_back(std::get<0>(op) ? 1 : 0);
      peer.push_back(p);
      msg.push_back(t.data_ptr());
      nbytes.push_back(n);
    }
    if (msg.empty()) return;
    PeerPtrs b = to_ptrs(bufs); SignalPadsH s = to_sig(sigs);
    c10::cuda::CUDAGuard guard(std::get<1>(ops[0]).device());
    ck_cuda(b2_p2p_batch_launch(&b, &s, send.data(), peer.data(), msg.data(), nbytes.data(), (int)msg.size(), rank, world,
                                cur_stream()), what);
  }, py::arg("bufs"), py::arg("sigs"), py::arg("ops"), py::arg("rank"), py::arg("world"));
  m.def("allreduce_sgd", [](std::vector<unsigned long long> grads, std::vector<unsigned long long> sigs, torch::Tensor params,
                            torch::Tensor momentum, c10::optional<torch::Tensor> step, double lr, double mu, double scale,
                            int rank, int world, bool zero_grads, int64_t grad_stride, c10::optional<torch::Tensor> done_counter,
                            c10::optional<torch::Tensor> aux, std::vector<unsigned long long> inbox, bool wire_bf16,
                            py::object lr_schedule, double weight_decay, bool nesterov, py::object max_grad_norm,
                            c10::optional<torch::Tensor> clip_workspace, c10::optional<torch::Tensor> grad_norm_out) {
    check_world(rank, world, "allreduce_sgd");
    check_sgd_options(weight_decay, nesterov, mu, "allreduce_sgd");
    const float max_norm = check_max_grad_norm(max_grad_norm, "allreduce_sgd");
    TORCH_CHECK((int)grads.size() == world && (int)sigs.size() == world, "allreduce_sgd: one gradient bucket and one signal pad "
                "per rank, got ", grads.size(), " and ", sigs.size(), " for world ", world);
    check_cuda_contig(params, "params"); check_cuda_contig(momentum, "momentum");
    const b2::LrSchedule sched = to_sched(lr_schedule);
    TORCH_CHECK(inbox.empty() || (int)inbox.size() == world, "inbox: one pointer per rank (or none)");
    PeerPtrs ib = to_ptrs(inbox);
    TORCH_CHECK(params.scalar_type() == torch::kFloat32 && momentum.scalar_type() == torch::kFloat32, "fp32 flat buffers");
    TORCH_CHECK(params.numel() % 4 == 0 && params.numel() == momentum.numel(), "flat buffers must be padded to 4 elements");
    PeerPtrs g = to_ptrs(grads); SignalPadsH s = to_sig(sigs);
    unsigned long long* st = step.has_value() ? reinterpret_cast<unsigned long long*>(step->data_ptr()) : nullptr;
    unsigned int* dc = done_counter.has_value() ? reinterpret_cast<unsigned int*>(done_counter->data_ptr()) : nullptr;
    TORCH_CHECK(st == nullptr || dc != nullptr, "a step counter needs a done_counter scratch word");
    float* ax = nullptr;
    if (aux.has_value()) { TORCH_CHECK(aux->is_cuda() && aux->scalar_type() == torch::kFloat32 && aux->numel() >= 13000); ax = aux->data_ptr<float>(); }
    float* ws = clip_ws_ptr(max_norm, clip_workspace, params.numel(), "allreduce_sgd");
    float* gn = grad_norm_ptr(grad_norm_out, "allreduce_sgd");
    c10::cuda::CUDAGuard guard(params.device());
    ck_cuda(b2_allreduce_sgd_launch(&g, &s, params.data_ptr<float>(), momentum.data_ptr<float>(), st, (size_t)params.numel(),
                                    (float)lr, (float)mu, (float)scale, rank, world, zero_grads, grad_stride, dc, ax,
                                    inbox.empty() ? nullptr : &ib, nullptr, nullptr, wire_bf16 ? 1 : 0, &sched, (float)weight_decay,
                                    nesterov ? 1 : 0, max_norm, ws, gn, cur_stream()),
            "allreduce_sgd launch");
  }, py::arg("grads"), py::arg("sigs"), py::arg("params"), py::arg("momentum"), py::arg("step"), py::arg("lr"), py::arg("mu"),
     py::arg("scale"), py::arg("rank"), py::arg("world"), py::arg("zero_grads"), py::arg("grad_stride") = 0,
     py::arg("done_counter") = py::none(), py::arg("aux") = py::none(), py::arg("inbox") = std::vector<unsigned long long>(),
     py::arg("wire_bf16") = false, py::arg("lr_schedule") = py::none(), py::arg("weight_decay") = 0.0, py::arg("nesterov") = false,
     py::arg("max_grad_norm") = py::none(), py::arg("clip_workspace") = py::none(), py::arg("grad_norm_out") = py::none());
  m.def("clip_workspace_numel", [](int64_t n) { return (int64_t)b2_clip_ws_floats((size_t)n); },
        "elements of the fp32 clip_workspace the optimizer kernels need for n flat parameters with max_grad_norm set");
  m.def("bn_launch", &bn_launch, py::arg("kind"), py::arg("x"), py::arg("dy"), py::arg("out"), py::arg("ex"), py::arg("stats"),
        py::arg("tickets"), py::arg("weight"), py::arg("bias"), py::arg("running_mean"), py::arg("running_var"),
        py::arg("num_batches_tracked"), py::arg("grad_weight"), py::arg("grad_bias"), py::arg("momentum"), py::arg("eps"),
        py::arg("max_blocks"), "one SyncBatchNorm kernel (csrc/batchnorm.cu); parallel/sync_bn.py drives them");
  m.def("grad_sqnorm_workspace_numel", [] { return b2_grad_sqnorm_ws_floats(); });
  m.def("grad_sqnorm", [](torch::Tensor g, torch::Tensor sqnorms, int k, torch::Tensor workspace,
                          c10::optional<torch::Tensor> grad_scale) {
    // sqnorms[k] = the sum of squares of g (fp32 per thread and CTA, fp64 across the CTAs in CTA order), for sgd_flat's clipping
    check_cuda_contig(g, "g"); check_cuda_contig(sqnorms, "sqnorms"); check_cuda_contig(workspace, "workspace");
    TORCH_CHECK(g.scalar_type() == torch::kFloat32 && (uintptr_t)g.data_ptr() % 16 == 0, "grad_sqnorm: g: 16-byte aligned fp32");
    TORCH_CHECK(sqnorms.scalar_type() == torch::kFloat64 && k >= 0 && k < sqnorms.numel(), "grad_sqnorm: sqnorms: fp64 with slot k");
    TORCH_CHECK(workspace.scalar_type() == torch::kFloat32 && workspace.numel() >= b2_grad_sqnorm_ws_floats(),
                "grad_sqnorm: workspace: fp32 [grad_sqnorm_workspace_numel()], zero before its first use");
    c10::cuda::CUDAGuard guard(g.device());
    const float* gs = amp_scalar_ptr(grad_scale, g, "grad_sqnorm", "grad_scale");
    ck_cuda(b2_grad_sqnorm_launch(g.data_ptr<float>(), (size_t)g.numel(), workspace.data_ptr<float>(), sqnorms.data_ptr<double>(), k,
                                  gs, cur_stream()), "grad_sqnorm launch");
  }, py::arg("g"), py::arg("sqnorms"), py::arg("k"), py::arg("workspace"), py::arg("grad_scale") = py::none());
  // FlatSGD's update of one fp32 bucket (csrc/sgd.cu): sgd_flat with lr / weight_decay, sgd_flat_grouped with group_map and
  // the groups' lrs / weight_decays (parameter vector i takes those of group group_map[i]), sgd_flat_cap with the scalars
  // from the block (with group_map, every group's).  With max_grad_norm, g is first scaled by the clip coefficient of the
  // norm of grad_sqnorm's per-bucket sums; with grad_scale, first unscaled.
  auto sgd_flat = [](const char* what, torch::Tensor& p, torch::Tensor& mom, torch::Tensor& g,
                     const c10::optional<torch::Tensor>& group_map, const std::vector<double>& lrs,
                     const std::vector<double>& weight_decays, const torch::Tensor* block, double mu, bool zero_grad, bool nesterov,
                     const py::object& max_grad_norm, const c10::optional<torch::Tensor>& sqnorms,
                     const c10::optional<torch::Tensor>& grad_norm_out, const c10::optional<torch::Tensor>& grad_scale,
                     const c10::optional<torch::Tensor>& found_inf) {
    // every group's weight decay (none: the capturable form's come from the block), checked through the smallest
    check_sgd_options(weight_decays.empty() ? 0.0 : *std::min_element(weight_decays.begin(), weight_decays.end()), nesterov, mu,
                      what);
    const Clip c = clip_args(max_grad_norm, sqnorms, grad_norm_out, what);
    const auto [gsc, fi] = amp_pair(grad_scale, found_inf, block != nullptr, p, what);
    check_flats({&p, &mom, &g}, p.numel(), false, "p, m and g", what);
    const int64_t n_ids = (p.numel() + 3) / 4;
    c10::cuda::CUDAGuard guard(p.device());
    if (block != nullptr) {
      ck_cuda(b2_sgd_flat_cap_launch(p.data_ptr<float>(), mom.data_ptr<float>(), g.data_ptr<float>(), (size_t)p.numel(),
                                     flat_map(group_map, n_ids, what), flat_block(*block, p, what), (float)mu, zero_grad ? 1 : 0,
                                     nesterov ? 1 : 0, c.max_norm, c.sq, c.n_buckets, c.gn, gsc, fi, cur_stream()),
              what);
    } else if (group_map.has_value()) {
      b2::SgdGroups gs;
      memset(&gs, 0, sizeof(gs));
      const int n_groups = check_groups(*group_map, n_ids, lrs, weight_decays, gs.lr, gs.wd, what);
      ck_cuda(b2_sgd_flat_grouped_launch(p.data_ptr<float>(), mom.data_ptr<float>(), g.data_ptr<float>(), (size_t)p.numel(),
                                         group_map->data_ptr<uint8_t>(), &gs, n_groups, (float)mu, zero_grad ? 1 : 0,
                                         nesterov ? 1 : 0, c.max_norm, c.sq, c.n_buckets, c.gn, gsc, cur_stream()),
              what);
    } else {
      ck_cuda(b2_sgd_flat_launch(p.data_ptr<float>(), mom.data_ptr<float>(), g.data_ptr<float>(), (size_t)p.numel(), (float)lrs[0],
                                 (float)mu, (float)weight_decays[0], zero_grad ? 1 : 0, nesterov ? 1 : 0, c.max_norm, c.sq,
                                 c.n_buckets, c.gn, gsc, cur_stream()),
              what);
    }
  };
  m.def("sgd_flat", [sgd_flat](torch::Tensor p, torch::Tensor mom, torch::Tensor g, double lr, double mu, double wd, bool zero_grad,
                               bool nesterov, py::object max_grad_norm, c10::optional<torch::Tensor> sqnorms,
                               c10::optional<torch::Tensor> grad_norm_out, c10::optional<torch::Tensor> grad_scale) {
    sgd_flat("sgd_flat", p, mom, g, c10::nullopt, {lr}, {wd}, nullptr, mu, zero_grad, nesterov, max_grad_norm, sqnorms,
             grad_norm_out, grad_scale, c10::nullopt);
  }, py::arg("p"), py::arg("m"), py::arg("g"), py::arg("lr"), py::arg("mu"), py::arg("weight_decay"), py::arg("zero_grad"),
     py::arg("nesterov") = false, py::arg("max_grad_norm") = py::none(), py::arg("sqnorms") = py::none(),
     py::arg("grad_norm_out") = py::none(), py::arg("grad_scale") = py::none());
  m.def("sgd_flat_grouped", [sgd_flat](torch::Tensor p, torch::Tensor mom, torch::Tensor g, torch::Tensor group_map,
                                       std::vector<double> lrs, std::vector<double> weight_decays, double mu, bool zero_grad,
                                       bool nesterov, py::object max_grad_norm, c10::optional<torch::Tensor> sqnorms,
                                       c10::optional<torch::Tensor> grad_norm_out, c10::optional<torch::Tensor> grad_scale) {
    sgd_flat("sgd_flat_grouped", p, mom, g, group_map, lrs, weight_decays, nullptr, mu, zero_grad, nesterov, max_grad_norm, sqnorms,
             grad_norm_out, grad_scale, c10::nullopt);
  }, py::arg("p"), py::arg("m"), py::arg("g"), py::arg("group_map"), py::arg("lrs"), py::arg("weight_decays"), py::arg("mu"),
     py::arg("zero_grad"), py::arg("nesterov") = false, py::arg("max_grad_norm") = py::none(), py::arg("sqnorms") = py::none(),
     py::arg("grad_norm_out") = py::none(), py::arg("grad_scale") = py::none());
  m.def("sgd_flat_cap", [sgd_flat](torch::Tensor p, torch::Tensor mom, torch::Tensor g, c10::optional<torch::Tensor> group_map,
                                   torch::Tensor block, double mu, bool zero_grad, bool nesterov, py::object max_grad_norm,
                                   c10::optional<torch::Tensor> sqnorms, c10::optional<torch::Tensor> grad_norm_out,
                                   c10::optional<torch::Tensor> grad_scale, c10::optional<torch::Tensor> found_inf) {
    sgd_flat("sgd_flat_cap", p, mom, g, group_map, {}, {}, &block, mu, zero_grad, nesterov, max_grad_norm, sqnorms, grad_norm_out,
             grad_scale, found_inf);
  }, py::arg("p"), py::arg("m"), py::arg("g"), py::arg("group_map"), py::arg("block"), py::arg("mu"), py::arg("zero_grad"),
     py::arg("nesterov") = false, py::arg("max_grad_norm") = py::none(), py::arg("sqnorms") = py::none(),
     py::arg("grad_norm_out") = py::none(), py::arg("grad_scale") = py::none(), py::arg("found_inf") = py::none());
  // FlatAdamW's update of one fp32 bucket (csrc/adamw.cu): adamw_flat with `scalars`, adamw_flat_grouped with group_map and
  // the groups' decays / step_sizes (1 - lr_g*wd_g and lr_g / (1 - beta1^t), fp64, each rounded once to fp32 here; the decay
  // and step_size of `scalars` are then not used), adamw_flat_cap with the scalars from the block (with group_map, every
  // group's).  Clipping and grad_scale as sgd_flat's.
  auto adamw_flat = [](const char* what, torch::Tensor& p, torch::Tensor& exp_avg, torch::Tensor& exp_avg_sq, torch::Tensor& g,
                       const c10::optional<torch::Tensor>& group_map, const std::vector<double>* scalars,
                       const std::vector<double>& decays, const std::vector<double>& step_sizes, const torch::Tensor* block,
                       bool zero_grad, const py::object& max_grad_norm, const c10::optional<torch::Tensor>& sqnorms,
                       const c10::optional<torch::Tensor>& grad_norm_out, const c10::optional<torch::Tensor>& grad_scale,
                       const c10::optional<torch::Tensor>& found_inf) {
    const b2::AdamwScalars sc = scalars != nullptr ? to_adamw(*scalars, what) : b2::AdamwScalars{};
    const Clip c = clip_args(max_grad_norm, sqnorms, grad_norm_out, what);
    const auto [gsc, fi] = amp_pair(grad_scale, found_inf, block != nullptr, p, what);
    check_flats({&p, &exp_avg, &exp_avg_sq, &g}, p.numel(), false, "p, exp_avg, exp_avg_sq and g", what);
    const int64_t n_ids = (p.numel() + 3) / 4;
    c10::cuda::CUDAGuard guard(p.device());
    if (block != nullptr) {
      ck_cuda(b2_adamw_flat_cap_launch(p.data_ptr<float>(), exp_avg.data_ptr<float>(), exp_avg_sq.data_ptr<float>(),
                                       g.data_ptr<float>(), (size_t)p.numel(), flat_map(group_map, n_ids, what),
                                       flat_block(*block, p, what), zero_grad ? 1 : 0, c.max_norm, c.sq, c.n_buckets, c.gn, gsc, fi,
                                       cur_stream()),
              what);
    } else if (group_map.has_value()) {
      b2::AdamwGroups gs;
      memset(&gs, 0, sizeof(gs));
      const int n_groups = check_groups(*group_map, n_ids, decays, step_sizes, gs.decay, gs.step_size, what);
      ck_cuda(b2_adamw_flat_grouped_launch(p.data_ptr<float>(), exp_avg.data_ptr<float>(), exp_avg_sq.data_ptr<float>(),
                                           g.data_ptr<float>(), (size_t)p.numel(), group_map->data_ptr<uint8_t>(), &sc, &gs,
                                           n_groups, zero_grad ? 1 : 0, c.max_norm, c.sq, c.n_buckets, c.gn, gsc, cur_stream()),
              what);
    } else {
      ck_cuda(b2_adamw_flat_launch(p.data_ptr<float>(), exp_avg.data_ptr<float>(), exp_avg_sq.data_ptr<float>(), g.data_ptr<float>(),
                                   (size_t)p.numel(), &sc, zero_grad ? 1 : 0, c.max_norm, c.sq, c.n_buckets, c.gn, gsc, cur_stream()),
              what);
    }
  };
  m.def("adamw_flat", [adamw_flat](torch::Tensor p, torch::Tensor exp_avg, torch::Tensor exp_avg_sq, torch::Tensor g,
                                   std::vector<double> scalars, bool zero_grad, py::object max_grad_norm,
                                   c10::optional<torch::Tensor> sqnorms, c10::optional<torch::Tensor> grad_norm_out,
                                   c10::optional<torch::Tensor> grad_scale) {
    adamw_flat("adamw_flat", p, exp_avg, exp_avg_sq, g, c10::nullopt, &scalars, {}, {}, nullptr, zero_grad, max_grad_norm, sqnorms,
               grad_norm_out, grad_scale, c10::nullopt);
  }, py::arg("p"), py::arg("exp_avg"), py::arg("exp_avg_sq"), py::arg("g"), py::arg("scalars"), py::arg("zero_grad"),
     py::arg("max_grad_norm") = py::none(), py::arg("sqnorms") = py::none(), py::arg("grad_norm_out") = py::none(),
     py::arg("grad_scale") = py::none());
  m.def("adamw_flat_grouped", [adamw_flat](torch::Tensor p, torch::Tensor exp_avg, torch::Tensor exp_avg_sq, torch::Tensor g,
                                           torch::Tensor group_map, std::vector<double> scalars, std::vector<double> decays,
                                           std::vector<double> step_sizes, bool zero_grad, py::object max_grad_norm,
                                           c10::optional<torch::Tensor> sqnorms, c10::optional<torch::Tensor> grad_norm_out,
                                           c10::optional<torch::Tensor> grad_scale) {
    adamw_flat("adamw_flat_grouped", p, exp_avg, exp_avg_sq, g, group_map, &scalars, decays, step_sizes, nullptr, zero_grad,
               max_grad_norm, sqnorms, grad_norm_out, grad_scale, c10::nullopt);
  }, py::arg("p"), py::arg("exp_avg"), py::arg("exp_avg_sq"), py::arg("g"), py::arg("group_map"), py::arg("scalars"),
     py::arg("decays"), py::arg("step_sizes"), py::arg("zero_grad"), py::arg("max_grad_norm") = py::none(),
     py::arg("sqnorms") = py::none(), py::arg("grad_norm_out") = py::none(), py::arg("grad_scale") = py::none());
  m.def("adamw_flat_cap", [adamw_flat](torch::Tensor p, torch::Tensor exp_avg, torch::Tensor exp_avg_sq, torch::Tensor g,
                                       c10::optional<torch::Tensor> group_map, torch::Tensor block, bool zero_grad,
                                       py::object max_grad_norm, c10::optional<torch::Tensor> sqnorms,
                                       c10::optional<torch::Tensor> grad_norm_out, c10::optional<torch::Tensor> grad_scale,
                                       c10::optional<torch::Tensor> found_inf) {
    adamw_flat("adamw_flat_cap", p, exp_avg, exp_avg_sq, g, group_map, nullptr, {}, {}, &block, zero_grad, max_grad_norm, sqnorms,
               grad_norm_out, grad_scale, found_inf);
  }, py::arg("p"), py::arg("exp_avg"), py::arg("exp_avg_sq"), py::arg("g"), py::arg("group_map"), py::arg("block"),
     py::arg("zero_grad"), py::arg("max_grad_norm") = py::none(), py::arg("sqnorms") = py::none(),
     py::arg("grad_norm_out") = py::none(), py::arg("grad_scale") = py::none(), py::arg("found_inf") = py::none());
  m.def("max_param_groups", [] { return b2::kMaxGroups; }, "the most parameter groups the grouped optimizer kernels take");
  // Capturable FlatSGD / FlatAdamW (csrc/flat_scalars.cuh): the layout of the scalar block in fp32 words and the byte sizes
  // of the block and the table
  m.def("flat_scalars_layout", [] {
    py::dict d;
    d["lr"] = offsetof(b2::FlatScalars, lr) / 4;
    d["wd"] = offsetof(b2::FlatScalars, wd) / 4;
    d["adamw"] = offsetof(b2::FlatScalars, adamw) / 4;
    d["sgd_lr"] = (offsetof(b2::FlatScalars, sgd) + offsetof(b2::SgdGroups, lr)) / 4;
    d["sgd_wd"] = (offsetof(b2::FlatScalars, sgd) + offsetof(b2::SgdGroups, wd)) / 4;
    d["decay"] = (offsetof(b2::FlatScalars, adamw_groups) + offsetof(b2::AdamwGroups, decay)) / 4;
    d["step_size"] = (offsetof(b2::FlatScalars, adamw_groups) + offsetof(b2::AdamwGroups, step_size)) / 4;
    d["block_bytes"] = sizeof(b2::FlatScalars);
    d["table_bytes"] = sizeof(b2::FlatHyper);
    return d;
  });
  // Upload the hyper-parameters (every group's base lr and weight decay in fp64, the AdamW constants, the schedule) and, with
  // `steps`, the step counter, then fill the block of the update run at the counter's value.  The values are staged in a
  // pinned buffer of torch's caching host allocator and copied with non_blocking copies (the allocator keeps the buffer until
  // the copy has run), so the call does not wait for the device.  Refused while the current stream is being captured: a
  // graph would replay this call's values.
  m.def("flat_scalars_sync", [](torch::Tensor table, torch::Tensor counter, torch::Tensor block, std::vector<double> lrs,
                                std::vector<double> weight_decays, double beta1, double beta2, double eps, py::object schedule,
                                c10::optional<int64_t> steps) {
    const FlatState st = flat_state(table, counter, block, "flat_scalars_sync");
    TORCH_CHECK(!lrs.empty() && lrs.size() <= (size_t)b2::kMaxGroups && lrs.size() == weight_decays.size(),
                "flat_scalars_sync: 1..", b2::kMaxGroups, " groups with one lr and one weight_decay each");
    TORCH_CHECK(!steps.has_value() || *steps >= 0, "flat_scalars_sync: steps must be >= 0");
    b2::FlatHyper h;
    std::memset(&h, 0, sizeof(h));
    h.sched = to_sched(schedule);
    h.beta1 = beta1; h.beta2 = beta2; h.eps = eps;
    h.n_groups = (int)lrs.size();
    for (size_t i = 0; i < lrs.size(); ++i) {
      TORCH_CHECK(std::isfinite((float)lrs[i]) && weight_decays[i] >= 0.0 && std::isfinite(weight_decays[i]),
                  "flat_scalars_sync: lr must be finite in fp32 and weight_decay finite and >= 0");
      h.lr[i] = lrs[i];
      h.wd[i] = weight_decays[i];
    }
    c10::cuda::CUDAGuard guard(counter.device());
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    ck_cuda((int)cudaStreamIsCapturing(cur_stream(), &cap), "flat_scalars_sync");
    TORCH_CHECK(cap == cudaStreamCaptureStatusNone, "flat_scalars_sync: the current stream is being captured; upload the "
                "hyper-parameters or set the step counter outside the capture");
    const int64_t nh = (int64_t)sizeof(b2::FlatHyper);
    auto staged = torch::empty({nh + 8}, torch::TensorOptions().dtype(torch::kUInt8).pinned_memory(true));
    std::memcpy(staged.data_ptr(), &h, sizeof(h));
    table.narrow(0, 0, nh).copy_(staged.narrow(0, 0, nh), /*non_blocking=*/true);
    if (steps.has_value()) {
      const unsigned long long s = (unsigned long long)*steps;
      std::memcpy(staged.data_ptr<uint8_t>() + nh, &s, sizeof(s));
      counter.view(torch::kUInt8).copy_(staged.narrow(0, nh, 8), /*non_blocking=*/true);
    }
    ck_cuda(b2_flat_scalars_launch(st.table, st.counter, st.block, 0, nullptr, cur_stream()), "flat_scalars_sync launch");
  }, py::arg("table"), py::arg("counter"), py::arg("block"), py::arg("lrs"), py::arg("weight_decays"), py::arg("beta1") = 0.0,
     py::arg("beta2") = 0.0, py::arg("eps") = 0.0, py::arg("schedule") = py::none(), py::arg("steps") = py::none());
  // counter += 1 and the block of the next update, in one single-CTA launch (advance = false: the block only).  found_inf
  // (GradScaler's, fp32 CUDA [1]): the gated advance, which leaves counter and block untouched when *found_inf != 0
  m.def("flat_scalars_advance", [](torch::Tensor table, torch::Tensor counter, torch::Tensor block, bool advance,
                                   c10::optional<torch::Tensor> found_inf) {
    const FlatState st = flat_state(table, counter, block, "flat_scalars_advance");
    const float* fi = amp_scalar_ptr(found_inf, counter, "flat_scalars_advance", "found_inf");
    TORCH_CHECK(fi == nullptr || advance, "flat_scalars_advance: found_inf gates an advance; it needs advance=True");
    c10::cuda::CUDAGuard guard(counter.device());
    ck_cuda(b2_flat_scalars_launch(st.table, st.counter, st.block, advance ? 1 : 0, fi, cur_stream()), "flat_scalars_advance launch");
  }, py::arg("table"), py::arg("counter"), py::arg("block"), py::arg("advance") = true, py::arg("found_inf") = py::none());
  // FlatEMA (csrc/ema.h): the entry table of (EMA array, live array) pairs, as (device table, host table); int64 rows of 8 words
  m.def("ema_table", [](const std::vector<torch::Tensor>& emas, const std::vector<torch::Tensor>& lives) {
    TORCH_CHECK(!emas.empty() && emas.size() == lives.size() && emas.size() < (size_t)INT32_MAX,
                "ema_table: one live tensor per EMA tensor, at least one pair");
    const torch::Device dev = emas[0].device();
    auto host = torch::zeros({(int64_t)emas.size() * 8}, torch::dtype(torch::kInt64));
    b2::EmaEntry* rows = reinterpret_cast<b2::EmaEntry*>(host.data_ptr<int64_t>());
    long long n_vec = 0, n_scalar = 0;
    for (size_t i = 0; i < emas.size(); ++i) {
      const torch::Tensor& e = emas[i];
      const torch::Tensor& p = lives[i];
      for (const auto* t : {&e, &p})
        TORCH_CHECK(t->is_cuda() && t->is_contiguous() && t->scalar_type() == torch::kFloat32 && t->device() == dev &&
                    t->numel() >= 1 && t->data_ptr() != nullptr, "ema_table: entry ", i, ": non-empty contiguous fp32 CUDA tensors "
                    "on one device");
      TORCH_CHECK(e.numel() == p.numel(), "ema_table: entry ", i, ": the EMA and the live tensor differ in size");
      const uintptr_t ea = (uintptr_t)e.data_ptr(), pa = (uintptr_t)p.data_ptr();
      b2::EmaEntry& r = rows[i];
      r.ema = e.data_ptr<float>();
      r.live = p.data_ptr<float>();
      r.n = e.numel();
      if (ea % 16 == pa % 16) {        // both reach a 16-byte boundary after the same number of elements
        r.head = std::min<long long>(r.n, (long long)((16 - ea % 16) % 16 / 4));
        r.n_vec = (r.n - r.head) / 4;
      } else {
        r.head = r.n;
        r.n_vec = 0;
      }
      r.vec_begin = n_vec;
      r.scalar_begin = n_scalar;
      n_vec += r.n_vec;
      n_scalar += r.n - 4 * r.n_vec;
    }
    return py::make_tuple(host.to(dev), host);
  }, py::arg("emas"), py::arg("lives"));
  // One launch over every entry: host-decided (counter None: copy, or lerp with w) or device-counter (counter: the optimizer's
  // int64 [1] step counter t; skip when t % every != 0, copy when t - every <= warmup_steps, lerp otherwise)
  m.def("ema_update", [](torch::Tensor table, torch::Tensor host, double w, bool copy, c10::optional<torch::Tensor> counter,
                         int64_t every, int64_t warmup_steps) {
    TORCH_CHECK(!host.is_cuda() && host.is_contiguous() && host.scalar_type() == torch::kInt64 && host.numel() >= 8 &&
                host.numel() % 8 == 0, "ema_update: host: the CPU int64 table from ema_table");
    TORCH_CHECK(table.is_cuda() && table.is_contiguous() && table.scalar_type() == torch::kInt64 && table.numel() == host.numel(),
                "ema_update: table: the CUDA int64 table from ema_table");
    TORCH_CHECK(every >= 1 && warmup_steps >= 0, "ema_update: every must be >= 1 and warmup_steps >= 0, got ", every, " and ",
                warmup_steps);
    TORCH_CHECK(std::isfinite(w) && w >= 0.0 && w <= 1.0, "ema_update: w = 1 - decay must be in [0, 1], got ", w);
    const int n = (int)(host.numel() / 8);
    const b2::EmaEntry* rows = reinterpret_cast<const b2::EmaEntry*>(host.data_ptr<int64_t>());
    for (int i = 0; i < n; ++i)
      TORCH_CHECK(rows[i].ema != nullptr && rows[i].live != nullptr && rows[i].n >= 1, "ema_update: entry ", i, " is empty");
    const long long n_vec = rows[n - 1].vec_begin + rows[n - 1].n_vec;
    const long long n_scalar = rows[n - 1].scalar_begin + rows[n - 1].n - 4 * rows[n - 1].n_vec;
    const long long* ctr = nullptr;
    if (counter.has_value()) {
      TORCH_CHECK(counter->is_cuda() && counter->scalar_type() == torch::kInt64 && counter->numel() == 1 &&
                  counter->device() == table.device(), "ema_update: counter: int64 CUDA [1] on the table's device");
      ctr = reinterpret_cast<const long long*>(counter->data_ptr<int64_t>());
    }
    c10::cuda::CUDAGuard guard(table.device());
    ck_cuda(b2_ema_launch(reinterpret_cast<const b2::EmaEntry*>(table.data_ptr<int64_t>()), n, n_vec, n_scalar, (float)w,
                          copy ? b2::EMA_COPY : b2::EMA_LERP, ctr, every, warmup_steps, cur_stream()),
            "ema_update launch");
  }, py::arg("table"), py::arg("host"), py::arg("w"), py::arg("copy") = false, py::arg("counter") = py::none(),
     py::arg("every") = 1, py::arg("warmup_steps") = 0);
  // FlatRMSprop's update of one fp32 bucket (csrc/rmsprop.cu).  scalars (fp64, each rounded once to fp32): (lr, weight_decay,
  // alpha, 1 - alpha, eps, momentum); grad_avg with centered, momentum_buffer with momentum > 0.  With max_grad_norm, g is
  // first scaled by the clip coefficient of the norm of grad_sqnorm's per-bucket sums; with grad_scale, first unscaled.
  // group_map (rmsprop_flat_grouped: lrs / weight_decays per group, rmsprop_flat_cap: from the block) picks each parameter
  // vector's lr and weight decay, which scalars then do not give.
  auto rmsprop_flat = [](const char* what, torch::Tensor& p, torch::Tensor& square_avg, const c10::optional<torch::Tensor>& grad_avg,
                         const c10::optional<torch::Tensor>& momentum_buffer, torch::Tensor& g,
                         const c10::optional<torch::Tensor>& group_map, const std::vector<double>* lrs,
                         const std::vector<double>* weight_decays, const torch::Tensor* block, const std::vector<double>& scalars,
                         bool centered, bool zero_grad, const py::object& max_grad_norm, const c10::optional<torch::Tensor>& sqnorms,
                         const c10::optional<torch::Tensor>& grad_norm_out, const c10::optional<torch::Tensor>& grad_scale,
                         const c10::optional<torch::Tensor>& found_inf) {
    const b2::RmspropScalars sc = to_rmsprop(scalars, centered, what);
    if (weight_decays != nullptr)
      for (double wd : *weight_decays) TORCH_CHECK(wd >= 0.0, what, ": weight_decay must be >= 0, got ", wd);
    const Clip c = clip_args(max_grad_norm, sqnorms, grad_norm_out, what);
    const auto [gsc, fi] = amp_pair(grad_scale, found_inf, block != nullptr, p, what);
    const auto opt = rmsprop_state({&p, &g}, square_avg, grad_avg, momentum_buffer, sc, p.numel(), false,
                                   "p, g, square_avg, grad_avg and momentum_buffer", what);
    const uint8_t* map = flat_map(group_map, (p.numel() + 3) / 4, what);
    b2::SgdGroups gs;
    memset(&gs, 0, sizeof(gs));
    const int n_groups = lrs != nullptr ? check_groups(*group_map, (p.numel() + 3) / 4, *lrs, *weight_decays, gs.lr, gs.wd, what) : 0;
    const b2::FlatScalars* blk = block != nullptr ? flat_block(*block, p, what) : nullptr;
    c10::cuda::CUDAGuard guard(p.device());
    ck_cuda(b2_rmsprop_flat_launch(p.data_ptr<float>(), square_avg.data_ptr<float>(), opt.first, opt.second, g.data_ptr<float>(),
                                   (size_t)p.numel(), map, &sc, &gs, n_groups, blk, zero_grad ? 1 : 0, c.max_norm, c.sq, c.n_buckets,
                                   c.gn, gsc, fi, cur_stream()),
            what);
  };
  m.def("rmsprop_flat", [rmsprop_flat](torch::Tensor p, torch::Tensor square_avg, c10::optional<torch::Tensor> grad_avg,
                                       c10::optional<torch::Tensor> momentum_buffer, torch::Tensor g, std::vector<double> scalars,
                                       bool centered, bool zero_grad, py::object max_grad_norm, c10::optional<torch::Tensor> sqnorms,
                                       c10::optional<torch::Tensor> grad_norm_out, c10::optional<torch::Tensor> grad_scale) {
    rmsprop_flat("rmsprop_flat", p, square_avg, grad_avg, momentum_buffer, g, c10::nullopt, nullptr, nullptr, nullptr, scalars,
                 centered, zero_grad, max_grad_norm, sqnorms, grad_norm_out, grad_scale, c10::nullopt);
  }, py::arg("p"), py::arg("square_avg"), py::arg("grad_avg"), py::arg("momentum_buffer"), py::arg("g"), py::arg("scalars"),
     py::arg("centered"), py::arg("zero_grad"), py::arg("max_grad_norm") = py::none(), py::arg("sqnorms") = py::none(),
     py::arg("grad_norm_out") = py::none(), py::arg("grad_scale") = py::none());
  m.def("rmsprop_flat_grouped", [rmsprop_flat](torch::Tensor p, torch::Tensor square_avg, c10::optional<torch::Tensor> grad_avg,
                                               c10::optional<torch::Tensor> momentum_buffer, torch::Tensor g, torch::Tensor group_map,
                                               std::vector<double> scalars, bool centered, std::vector<double> lrs,
                                               std::vector<double> weight_decays, bool zero_grad, py::object max_grad_norm,
                                               c10::optional<torch::Tensor> sqnorms, c10::optional<torch::Tensor> grad_norm_out,
                                               c10::optional<torch::Tensor> grad_scale) {
    rmsprop_flat("rmsprop_flat_grouped", p, square_avg, grad_avg, momentum_buffer, g, group_map, &lrs, &weight_decays, nullptr,
                 scalars, centered, zero_grad, max_grad_norm, sqnorms, grad_norm_out, grad_scale, c10::nullopt);
  }, py::arg("p"), py::arg("square_avg"), py::arg("grad_avg"), py::arg("momentum_buffer"), py::arg("g"), py::arg("group_map"),
     py::arg("scalars"), py::arg("centered"), py::arg("lrs"), py::arg("weight_decays"), py::arg("zero_grad"),
     py::arg("max_grad_norm") = py::none(), py::arg("sqnorms") = py::none(), py::arg("grad_norm_out") = py::none(),
     py::arg("grad_scale") = py::none());
  m.def("rmsprop_flat_cap", [rmsprop_flat](torch::Tensor p, torch::Tensor square_avg, c10::optional<torch::Tensor> grad_avg,
                                           c10::optional<torch::Tensor> momentum_buffer, torch::Tensor g,
                                           c10::optional<torch::Tensor> group_map, torch::Tensor block, std::vector<double> scalars,
                                           bool centered, bool zero_grad, py::object max_grad_norm,
                                           c10::optional<torch::Tensor> sqnorms, c10::optional<torch::Tensor> grad_norm_out,
                                           c10::optional<torch::Tensor> grad_scale, c10::optional<torch::Tensor> found_inf) {
    rmsprop_flat("rmsprop_flat_cap", p, square_avg, grad_avg, momentum_buffer, g, group_map, nullptr, nullptr, &block, scalars,
                 centered, zero_grad, max_grad_norm, sqnorms, grad_norm_out, grad_scale, found_inf);
  }, py::arg("p"), py::arg("square_avg"), py::arg("grad_avg"), py::arg("momentum_buffer"), py::arg("g"), py::arg("group_map"),
     py::arg("block"), py::arg("scalars"), py::arg("centered"), py::arg("zero_grad"), py::arg("max_grad_norm") = py::none(),
     py::arg("sqnorms") = py::none(), py::arg("grad_norm_out") = py::none(), py::arg("grad_scale") = py::none(),
     py::arg("found_inf") = py::none());
  // The sharded step of one bucket with RMSprop (csrc/sharded_sgd.cu, the RMSprop instances): as sharded_adamw, with this rank's
  // square_avg shard and, with centered / momentum > 0, its grad_avg / momentum_buffer shards.  sharded_rmsprop_grouped:
  // group_map holds this rank's ids and lrs / weight_decays the groups'; sharded_rmsprop_cap: lr and weight decay (with
  // group_map: every group's) from the block.
  auto sharded_rmsprop = [](const char* what, bool bf16, const std::vector<unsigned long long>& grads,
                            const std::vector<unsigned long long>& params, const std::vector<unsigned long long>& sigs,
                            torch::Tensor& square_avg, const c10::optional<torch::Tensor>& grad_avg,
                            const c10::optional<torch::Tensor>& momentum_buffer, const c10::optional<torch::Tensor>& group_map,
                            const std::vector<double>* lrs, const std::vector<double>* weight_decays, const torch::Tensor* block,
                            size_t n_vec, const std::vector<double>& scalars, bool centered, double scale, bool zero_grad, int rank,
                            int world, int max_blocks) {
    const Peers pr = sharded_peers(what, grads, params, nullptr, sigs, n_vec, bf16, rank, world);
    const b2::RmspropScalars sc = to_rmsprop(scalars, centered, what);
    if (weight_decays != nullptr)
      for (double wd : *weight_decays) TORCH_CHECK(wd >= 0.0, what, ": weight_decay must be >= 0, got ", wd);
    const auto opt = rmsprop_state({}, square_avg, grad_avg, momentum_buffer, sc, pr.shard, true,
                                   "square_avg, grad_avg and momentum_buffer (this rank's slice)", what);
    const uint8_t* map = flat_map(group_map, pr.shard / 4, what);
    b2::SgdGroups gs;
    memset(&gs, 0, sizeof(gs));
    const int n_groups = lrs != nullptr ? check_groups(*group_map, pr.shard / 4, *lrs, *weight_decays, gs.lr, gs.wd, what) : 0;
    c10::cuda::CUDAGuard guard(square_avg.device());
    if (block != nullptr) {
      const b2::FlatScalars* blk = flat_block(*block, square_avg, what);
      ck_cuda(b2_sharded_rmsprop_cap_launch(bf16 ? 1 : 0, &pr.grads, &pr.params, &pr.sigs, square_avg.data_ptr<float>(), opt.first,
                                            opt.second, map, blk, &sc, n_vec, (float)scale, zero_grad ? 1 : 0, rank, world, max_blocks,
                                            cur_stream()),
              what);
      return;
    }
    ck_cuda(b2_sharded_rmsprop_launch(bf16 ? 1 : 0, &pr.grads, &pr.params, &pr.sigs, square_avg.data_ptr<float>(), opt.first,
                                      opt.second, map, &sc, &gs, n_groups, n_vec, (float)scale, zero_grad ? 1 : 0, rank, world,
                                      max_blocks, cur_stream()),
            what);
  };
  m.def("sharded_rmsprop", [sharded_rmsprop](bool bf16, std::vector<unsigned long long> grads, std::vector<unsigned long long> params,
                                             std::vector<unsigned long long> sigs, torch::Tensor square_avg,
                                             c10::optional<torch::Tensor> grad_avg, c10::optional<torch::Tensor> momentum_buffer,
                                             size_t n_vec, std::vector<double> scalars, bool centered, double scale, bool zero_grad,
                                             int rank, int world, int max_blocks) {
    sharded_rmsprop("sharded_rmsprop", bf16, grads, params, sigs, square_avg, grad_avg, momentum_buffer, c10::nullopt, nullptr,
                    nullptr, nullptr, n_vec, scalars, centered, scale, zero_grad, rank, world, max_blocks);
  }, py::arg("bf16"), py::arg("grads"), py::arg("params"), py::arg("sigs"), py::arg("square_avg"), py::arg("grad_avg"),
     py::arg("momentum_buffer"), py::arg("n_vec"), py::arg("scalars"), py::arg("centered"), py::arg("scale"), py::arg("zero_grad"),
     py::arg("rank"), py::arg("world"), py::arg("max_blocks") = 0);
  m.def("sharded_rmsprop_grouped", [sharded_rmsprop](bool bf16, std::vector<unsigned long long> grads,
                                                     std::vector<unsigned long long> params, std::vector<unsigned long long> sigs,
                                                     torch::Tensor square_avg, c10::optional<torch::Tensor> grad_avg,
                                                     c10::optional<torch::Tensor> momentum_buffer, torch::Tensor group_map, size_t n_vec,
                                                     std::vector<double> scalars, bool centered, std::vector<double> lrs,
                                                     std::vector<double> weight_decays, double scale, bool zero_grad, int rank,
                                                     int world, int max_blocks) {
    sharded_rmsprop("sharded_rmsprop_grouped", bf16, grads, params, sigs, square_avg, grad_avg, momentum_buffer, group_map, &lrs,
                    &weight_decays, nullptr, n_vec, scalars, centered, scale, zero_grad, rank, world, max_blocks);
  }, py::arg("bf16"), py::arg("grads"), py::arg("params"), py::arg("sigs"), py::arg("square_avg"), py::arg("grad_avg"),
     py::arg("momentum_buffer"), py::arg("group_map"), py::arg("n_vec"), py::arg("scalars"), py::arg("centered"), py::arg("lrs"),
     py::arg("weight_decays"), py::arg("scale"), py::arg("zero_grad"), py::arg("rank"), py::arg("world"), py::arg("max_blocks") = 0);
  m.def("sharded_rmsprop_cap", [sharded_rmsprop](bool bf16, std::vector<unsigned long long> grads, std::vector<unsigned long long> params,
                                                 std::vector<unsigned long long> sigs, torch::Tensor square_avg,
                                                 c10::optional<torch::Tensor> grad_avg, c10::optional<torch::Tensor> momentum_buffer,
                                                 c10::optional<torch::Tensor> group_map, torch::Tensor block, size_t n_vec,
                                                 std::vector<double> scalars, bool centered, double scale, bool zero_grad, int rank,
                                                 int world, int max_blocks) {
    sharded_rmsprop("sharded_rmsprop_cap", bf16, grads, params, sigs, square_avg, grad_avg, momentum_buffer, group_map, nullptr,
                    nullptr, &block, n_vec, scalars, centered, scale, zero_grad, rank, world, max_blocks);
  }, py::arg("bf16"), py::arg("grads"), py::arg("params"), py::arg("sigs"), py::arg("square_avg"), py::arg("grad_avg"),
     py::arg("momentum_buffer"), py::arg("group_map"), py::arg("block"), py::arg("n_vec"), py::arg("scalars"), py::arg("centered"),
     py::arg("scale"), py::arg("zero_grad"), py::arg("rank"), py::arg("world"), py::arg("max_blocks") = 0);
  m.def("layerwise_chunk_elems", [] { return (int64_t)b2::kLwChunk; }, "the largest chunk of a layer-wise chunk table");
  m.def("layerwise_table", &layerwise_table, py::arg("offsets"), py::arg("numels"), py::arg("adapt"), py::arg("n"),
        py::arg("device"), "FlatLAMB / FlatLARS: (the chunk table of one bucket on `device`, its number of chunks)");
  m.def("lamb_flat", [](torch::Tensor p, torch::Tensor exp_avg, torch::Tensor exp_avg_sq, torch::Tensor g, torch::Tensor table,
                        int64_t n_chunks, torch::Tensor partials, torch::Tensor tickets, torch::Tensor sums, torch::Tensor ratios,
                        std::vector<double> scalars, bool zero_grad, py::object max_grad_norm,
                        c10::optional<torch::Tensor> sqnorms, c10::optional<torch::Tensor> grad_norm_out,
                        c10::optional<torch::Tensor> grad_scale) {
    // FlatLAMB's update of one fp32 bucket (csrc/layerwise.cu).  scalars (fp64, each rounded once to fp32 here):
    // (1 - beta1, beta2, 1 - beta2, sqrt(1 - beta2^t), eps, 1 / (1 - beta1^t), lr, weight_decay)
    TORCH_CHECK(scalars.size() == 8, "lamb_flat: scalars: (1 - beta1, beta2, 1 - beta2, sqrt(bc2), eps, 1 / bc1, lr, "
                "weight_decay), got ", scalars.size(), " values");
    for (double x : scalars) TORCH_CHECK(std::isfinite(x) && std::isfinite((float)x), "lamb_flat: scalars must be finite in fp32");
    TORCH_CHECK((float)scalars[3] > 0.f && scalars[4] >= 0.0, "lamb_flat: sqrt(bc2) must be > 0 (update t >= 1) and eps >= 0");
    b2::LwArgs a = layerwise_args("lamb_flat", p, g, {&exp_avg, &exp_avg_sq}, table, n_chunks, partials, tickets, sums, ratios,
                                  zero_grad, max_grad_norm, sqnorms, grad_norm_out, grad_scale);
    a.w1 = (float)scalars[0]; a.beta2 = (float)scalars[1]; a.c2 = (float)scalars[2]; a.sbc2 = (float)scalars[3];
    a.eps = (float)scalars[4]; a.rbc1 = (float)scalars[5]; a.lr = (float)scalars[6]; a.wd = (float)scalars[7];
    c10::cuda::CUDAGuard guard(p.device());
    ck_cuda(b2_layerwise_launch(1, &a, cur_stream()), "lamb_flat launch");
  }, py::arg("p"), py::arg("exp_avg"), py::arg("exp_avg_sq"), py::arg("g"), py::arg("table"), py::arg("n_chunks"),
     py::arg("partials"), py::arg("tickets"), py::arg("sums"), py::arg("ratios"), py::arg("scalars"), py::arg("zero_grad"),
     py::arg("max_grad_norm") = py::none(), py::arg("sqnorms") = py::none(), py::arg("grad_norm_out") = py::none(),
     py::arg("grad_scale") = py::none());
  m.def("lars_flat", [](torch::Tensor p, torch::Tensor momentum_buf, torch::Tensor g, torch::Tensor table, int64_t n_chunks,
                        torch::Tensor partials, torch::Tensor tickets, torch::Tensor sums, torch::Tensor ratios, double lr,
                        double momentum, double weight_decay, double trust_coefficient, double eps, bool nesterov, bool zero_grad,
                        py::object max_grad_norm, c10::optional<torch::Tensor> sqnorms, c10::optional<torch::Tensor> grad_norm_out,
                        c10::optional<torch::Tensor> grad_scale) {
    // FlatLARS's update of one fp32 bucket (csrc/layerwise.cu)
    check_sgd_options(weight_decay, nesterov, momentum, "lars_flat");
    TORCH_CHECK(std::isfinite(lr) && std::isfinite(momentum) && std::isfinite(weight_decay) && trust_coefficient > 0.0 &&
                std::isfinite(trust_coefficient) && eps >= 0.0 && std::isfinite(eps),
                "lars_flat: lr, momentum and weight_decay finite, trust_coefficient > 0 and eps >= 0 finite");
    b2::LwArgs a = layerwise_args("lars_flat", p, g, {&momentum_buf}, table, n_chunks, partials, tickets, sums, ratios, zero_grad,
                                  max_grad_norm, sqnorms, grad_norm_out, grad_scale);
    a.lr = (float)lr; a.mu = (float)momentum; a.wd = (float)weight_decay; a.nesterov = nesterov ? 1 : 0;
    a.eta64 = trust_coefficient; a.wd64 = weight_decay; a.eps64 = eps;
    c10::cuda::CUDAGuard guard(p.device());
    ck_cuda(b2_layerwise_launch(0, &a, cur_stream()), "lars_flat launch");
  }, py::arg("p"), py::arg("momentum_buffer"), py::arg("g"), py::arg("table"), py::arg("n_chunks"), py::arg("partials"),
     py::arg("tickets"), py::arg("sums"), py::arg("ratios"), py::arg("lr"), py::arg("momentum"), py::arg("weight_decay"),
     py::arg("trust_coefficient"), py::arg("eps"), py::arg("nesterov"), py::arg("zero_grad"),
     py::arg("max_grad_norm") = py::none(), py::arg("sqnorms") = py::none(), py::arg("grad_norm_out") = py::none(),
     py::arg("grad_scale") = py::none());
  py::class_<ShardedLwTable>(m, "ShardedLwTable", "one rank's chunk table of a sharded FlatLAMB / FlatLARS bucket")
      .def_readonly("table", &ShardedLwTable::table)
      .def_readonly("n_chunks", &ShardedLwTable::n_chunks)
      .def_readonly("n", &ShardedLwTable::n)
      .def_readonly("rank", &ShardedLwTable::rank)
      .def_readonly("world", &ShardedLwTable::world);
  m.def("sharded_layerwise_table", &sharded_layerwise_table, py::arg("offsets"), py::arg("numels"), py::arg("adapt"), py::arg("n"),
        py::arg("rank"), py::arg("world"), py::arg("device"),
        "sharded FlatLAMB / FlatLARS: the chunk table of rank `rank`'s slice of a padded bucket of n elements");
  // The sharded FlatLAMB update of one bucket (csrc/sharded_layerwise.cu): the gradient exchange, LAMB on this rank's slice
  // with its exp_avg / exp_avg_sq shards, the per-tensor sums exchanged through the symmetric `sums` buffers ([2 * tensors]
  // fp64 per rank), and the new parameters stored into every rank's flat in `params`.  scalars: lamb_flat's.
  m.def("sharded_lamb", [](bool bf16, std::vector<unsigned long long> grads, std::vector<unsigned long long> params,
                           std::vector<unsigned long long> sums, std::vector<unsigned long long> sigs, torch::Tensor exp_avg,
                           torch::Tensor exp_avg_sq, const ShardedLwTable& table, torch::Tensor partials,
                           torch::Tensor tickets, torch::Tensor ratios, size_t n_vec, std::vector<double> scalars, double scale,
                           bool zero_grad, int rank, int world, int max_blocks) {
    TORCH_CHECK(scalars.size() == 8, "sharded_lamb: scalars: (1 - beta1, beta2, 1 - beta2, sqrt(bc2), eps, 1 / bc1, lr, "
                "weight_decay), got ", scalars.size(), " values");
    for (double x : scalars) TORCH_CHECK(std::isfinite(x) && std::isfinite((float)x), "sharded_lamb: scalars must be finite in fp32");
    TORCH_CHECK((float)scalars[3] > 0.f && scalars[4] >= 0.0, "sharded_lamb: sqrt(bc2) must be > 0 (update t >= 1) and eps >= 0");
    auto [a, pr] = sharded_layerwise_args("sharded_lamb", true, bf16, grads, params, sums, sigs, {&exp_avg, &exp_avg_sq},
                                          table, partials, tickets, ratios, n_vec, zero_grad, rank, world);
    a.w1 = (float)scalars[0]; a.beta2 = (float)scalars[1]; a.c2 = (float)scalars[2]; a.sbc2 = (float)scalars[3];
    a.eps = (float)scalars[4]; a.rbc1 = (float)scalars[5]; a.lr = (float)scalars[6]; a.wd = (float)scalars[7];
    c10::cuda::CUDAGuard guard(exp_avg.device());
    ck_cuda(b2_sharded_layerwise_launch(1, bf16 ? 1 : 0, &pr.grads, &pr.params, &pr.sums, &pr.sigs, &a, n_vec, (float)scale, rank,
                                        world, max_blocks, cur_stream()), "sharded_lamb launch");
  }, py::arg("bf16"), py::arg("grads"), py::arg("params"), py::arg("sums"), py::arg("sigs"), py::arg("exp_avg"),
     py::arg("exp_avg_sq"), py::arg("table"), py::arg("partials"), py::arg("tickets"), py::arg("ratios"),
     py::arg("n_vec"), py::arg("scalars"), py::arg("scale"), py::arg("zero_grad"), py::arg("rank"), py::arg("world"),
     py::arg("max_blocks") = 0);
  // The sharded FlatLARS update: as sharded_lamb, with this rank's momentum shard and `grad_workspace`, a shard that keeps the
  // averaged gradient of the slice between the two kernels.
  m.def("sharded_lars", [](bool bf16, std::vector<unsigned long long> grads, std::vector<unsigned long long> params,
                           std::vector<unsigned long long> sums, std::vector<unsigned long long> sigs, torch::Tensor momentum_buf,
                           torch::Tensor grad_workspace, const ShardedLwTable& table, torch::Tensor partials,
                           torch::Tensor tickets, torch::Tensor ratios, size_t n_vec, double lr, double momentum,
                           double weight_decay, double trust_coefficient, double eps, bool nesterov, double scale, bool zero_grad,
                           int rank, int world, int max_blocks) {
    check_sgd_options(weight_decay, nesterov, momentum, "sharded_lars");
    TORCH_CHECK(std::isfinite(lr) && std::isfinite(momentum) && std::isfinite(weight_decay) && trust_coefficient > 0.0 &&
                std::isfinite(trust_coefficient) && eps >= 0.0 && std::isfinite(eps),
                "sharded_lars: lr, momentum and weight_decay finite, trust_coefficient > 0 and eps >= 0 finite");
    auto [a, pr] = sharded_layerwise_args("sharded_lars", false, bf16, grads, params, sums, sigs, {&momentum_buf, &grad_workspace},
                                          table, partials, tickets, ratios, n_vec, zero_grad, rank, world);
    a.lr = (float)lr; a.mu = (float)momentum; a.wd = (float)weight_decay; a.nesterov = nesterov ? 1 : 0;
    a.eta64 = trust_coefficient; a.wd64 = weight_decay; a.eps64 = eps;
    c10::cuda::CUDAGuard guard(momentum_buf.device());
    ck_cuda(b2_sharded_layerwise_launch(0, bf16 ? 1 : 0, &pr.grads, &pr.params, &pr.sums, &pr.sigs, &a, n_vec, (float)scale, rank,
                                        world, max_blocks, cur_stream()), "sharded_lars launch");
  }, py::arg("bf16"), py::arg("grads"), py::arg("params"), py::arg("sums"), py::arg("sigs"), py::arg("momentum_buffer"),
     py::arg("grad_workspace"), py::arg("table"), py::arg("partials"), py::arg("tickets"), py::arg("ratios"),
     py::arg("n_vec"), py::arg("lr"), py::arg("momentum"), py::arg("weight_decay"), py::arg("trust_coefficient"), py::arg("eps"),
     py::arg("nesterov"), py::arg("scale"), py::arg("zero_grad"), py::arg("rank"), py::arg("world"), py::arg("max_blocks") = 0);
  m.def("adafactor_chunk_elems", [] { return (int64_t)b2::kAfChunk; }, "the largest chunk of an Adafactor chunk table");
  m.def("adafactor_table", &adafactor_table, py::arg("offsets"), py::arg("shapes"), py::arg("strides"), py::arg("state_offsets"),
        py::arg("groups"), py::arg("n"), py::arg("n_state"), py::arg("n_groups"), py::arg("device"),
        "FlatAdafactor: (the chunk table of one bucket on `device`, chunks, row / column partials, row_var means)");
  m.def("adafactor_flat", [](torch::Tensor p, torch::Tensor state, torch::Tensor g, torch::Tensor table, int64_t n_chunks,
                             torch::Tensor partials, torch::Tensor rc, torch::Tensor means, torch::Tensor tickets, torch::Tensor alpha,
                             torch::Tensor step, std::vector<double> scalars, std::vector<double> rho, std::vector<double> decay,
                             bool zero_grad, py::object max_grad_norm, c10::optional<torch::Tensor> sqnorms,
                             c10::optional<torch::Tensor> grad_norm_out, c10::optional<torch::Tensor> grad_scale) {
    // FlatAdafactor's update of one fp32 bucket (csrc/adafactor.cu).  scalars (fp64): (t ** beta2_decay, eps1, eps2, d), the
    // first two rounded once to fp32 here, eps1^2 formed in fp64 and rounded once; per group rho_t (fp64) and
    // 1 - lr * weight_decay (rounded once to fp32).
    const char* what = "adafactor_flat";
    for (const torch::Tensor* t : {&p, &g, &state}) {
      check_cuda_contig(*t, what);
      TORCH_CHECK(t->scalar_type() == torch::kFloat32 && t->device() == p.device(), what,
                  ": parameters, gradients and state: contiguous fp32 CUDA on one device");
    }
    TORCH_CHECK(g.numel() == p.numel(), what, ": the gradient flat has ", g.numel(), " elements, the parameter flat ", p.numel());
    for (const torch::Tensor* t : {&table, &partials, &rc, &means, &tickets, &alpha, &step}) {
      check_cuda_contig(*t, what);
      TORCH_CHECK(t->device() == p.device(), what, ": the table and the workspaces live on the parameters' device");
    }
    const int64_t n_tensors = tickets.numel();
    TORCH_CHECK(n_chunks >= 1 && n_chunks <= p.numel() && n_tensors >= 1 && table.scalar_type() == torch::kInt64 &&
                table.numel() == n_chunks * b2::kAfChunkRow + n_tensors * b2::kAfTensorRow, what, ": table: int64 of chunks * ",
                b2::kAfChunkRow, " + tensors * ", b2::kAfTensorRow, " entries from adafactor_table, tickets: one per tensor");
    TORCH_CHECK(tickets.scalar_type() == torch::kInt32, what, ": tickets: int32 [tensors], zero before the first call");
    TORCH_CHECK(partials.scalar_type() == torch::kFloat32 && partials.numel() == 2 * n_chunks, what, ": partials: fp32 [2 * chunks]");
    TORCH_CHECK(rc.scalar_type() == torch::kFloat32 && means.scalar_type() == torch::kFloat32 && rc.numel() >= 1 && means.numel() >= 1,
                what, ": rc and means: fp32, as many as adafactor_table gives (at least one element each)");
    TORCH_CHECK(alpha.scalar_type() == torch::kFloat64 && alpha.numel() == n_tensors && step.scalar_type() == torch::kFloat32 &&
                step.numel() == n_tensors, what, ": alpha: fp64 [tensors], step: fp32 [tensors]");
    TORCH_CHECK(scalars.size() == 4, what, ": scalars: (t ** beta2_decay, eps1, eps2, d), got ", scalars.size(), " values");
    for (double x : scalars) TORCH_CHECK(std::isfinite(x) && std::isfinite((float)x), what, ": scalars must be finite in fp32");
    TORCH_CHECK(scalars[0] >= 0.0 && scalars[0] <= 1.0 && scalars[1] >= 0.0 && scalars[2] >= 0.0 && scalars[3] >= 1.0, what,
                ": t ** beta2_decay in [0, 1], eps1 >= 0, eps2 >= 0 and d >= 1");
    TORCH_CHECK(!rho.empty() && rho.size() <= (size_t)b2::kMaxGroups && rho.size() == decay.size(), what, ": 1..", b2::kMaxGroups,
                " groups with one rho and one decay each");
    b2::AfArgs a;
    std::memset(&a, 0, sizeof(a));
    a.p = p.data_ptr<float>(); a.g = g.data_ptr<float>(); a.state = state.data_ptr<float>();
    a.n = (size_t)p.numel();
    a.table = reinterpret_cast<const long long*>(table.data_ptr<int64_t>());
    a.n_chunks = (int)n_chunks; a.n_tensors = (int)n_tensors;
    a.partials = partials.data_ptr<float>(); a.rc = rc.data_ptr<float>(); a.means = means.data_ptr<float>();
    a.tickets = reinterpret_cast<unsigned int*>(tickets.data_ptr<int32_t>());
    a.alpha = alpha.data_ptr<double>(); a.step = step.data_ptr<float>();
    a.zero_grad = zero_grad ? 1 : 0;
    a.w = (float)scalars[0]; a.eps1 = (float)scalars[1]; a.eps1sq = (float)(scalars[1] * scalars[1]);
    a.eps2 = scalars[2]; a.d = scalars[3];
    a.n_groups = (int)rho.size();
    for (size_t i = 0; i < rho.size(); ++i) {
      TORCH_CHECK(std::isfinite(rho[i]) && rho[i] >= 0.0 && std::isfinite((float)decay[i]), what,
                  ": per-group rho must be finite and >= 0, decay finite in fp32");
      a.rho[i] = rho[i];
      a.decay[i] = (float)decay[i];
    }
    const Clip c = clip_args(max_grad_norm, sqnorms, grad_norm_out, what);
    a.max_norm = c.max_norm; a.sqnorms = c.sq; a.n_buckets = c.n_buckets; a.grad_norm_out = c.gn;
    a.grad_scale = amp_scalar_ptr(grad_scale, p, what, "grad_scale");
    c10::cuda::CUDAGuard guard(p.device());
    ck_cuda(b2_adafactor_launch(&a, cur_stream()), "adafactor_flat launch");
  }, py::arg("p"), py::arg("state"), py::arg("g"), py::arg("table"), py::arg("n_chunks"), py::arg("partials"), py::arg("rc"),
     py::arg("means"), py::arg("tickets"), py::arg("alpha"), py::arg("step"), py::arg("scalars"), py::arg("rho"), py::arg("decay"),
     py::arg("zero_grad"), py::arg("max_grad_norm") = py::none(), py::arg("sqnorms") = py::none(),
     py::arg("grad_norm_out") = py::none(), py::arg("grad_scale") = py::none());
  // Sharded optimizer step of one bucket (csrc/sharded_sgd.cu): reduce-scatter of the gradient buckets `grads`, momentum SGD on
  // this rank's slice with its momentum shard, and the new parameters stored into every rank's flat in `params`.  n_vec counts
  // the 16-byte vectors of one gradient bucket; raw per-rank pointers, like `allreduce`.  sharded_sgd takes lr / weight_decay,
  // sharded_sgd_grouped group_map (this rank's ids, one per fp32 parameter vector of its slice: n_vec / world x 1, x 2 with
  // bf16) and the groups' lrs / weight_decays, sharded_sgd_cap the scalars from the block (with group_map, every group's).
  auto sharded_sgd = [](const char* what, bool bf16, const std::vector<unsigned long long>& grads,
                        const std::vector<unsigned long long>& params, const std::vector<unsigned long long>& sigs,
                        torch::Tensor& momentum, const c10::optional<torch::Tensor>& group_map, const std::vector<double>& lrs,
                        const std::vector<double>& weight_decays, const torch::Tensor* block, size_t n_vec, double mu, bool nesterov,
                        double scale, bool zero_grad, int rank, int world, int max_blocks) {
    const Peers pr = sharded_peers(what, grads, params, nullptr, sigs, n_vec, bf16, rank, world);
    // every group's weight decay (none: the capturable form's come from the block), checked through the smallest
    check_sgd_options(weight_decays.empty() ? 0.0 : *std::min_element(weight_decays.begin(), weight_decays.end()), nesterov, mu,
                      what);
    check_flats({&momentum}, pr.shard, true, "momentum (this rank's slice)", what);
    c10::cuda::CUDAGuard guard(momentum.device());
    if (block != nullptr) {
      ck_cuda(b2_sharded_sgd_cap_launch(bf16 ? 1 : 0, &pr.grads, &pr.params, &pr.sigs, momentum.data_ptr<float>(),
                                        flat_map(group_map, pr.shard / 4, what), flat_block(*block, momentum, what), n_vec, (float)mu,
                                        nesterov ? 1 : 0, (float)scale, zero_grad ? 1 : 0, rank, world, max_blocks, cur_stream()),
              what);
    } else if (group_map.has_value()) {
      b2::SgdGroups gs;
      memset(&gs, 0, sizeof(gs));
      const int n_groups = check_groups(*group_map, pr.shard / 4, lrs, weight_decays, gs.lr, gs.wd, what);
      ck_cuda(b2_sharded_sgd_grouped_launch(bf16 ? 1 : 0, &pr.grads, &pr.params, &pr.sigs, momentum.data_ptr<float>(),
                                            group_map->data_ptr<uint8_t>(), &gs, n_groups, n_vec, (float)mu, nesterov ? 1 : 0,
                                            (float)scale, zero_grad ? 1 : 0, rank, world, max_blocks, cur_stream()),
              what);
    } else {
      ck_cuda(b2_sharded_sgd_launch(bf16 ? 1 : 0, &pr.grads, &pr.params, &pr.sigs, momentum.data_ptr<float>(), n_vec, (float)lrs[0],
                                    (float)mu, (float)weight_decays[0], nesterov ? 1 : 0, (float)scale, zero_grad ? 1 : 0, rank, world,
                                    max_blocks, cur_stream()),
              what);
    }
  };
  m.def("sharded_sgd", [sharded_sgd](bool bf16, std::vector<unsigned long long> grads, std::vector<unsigned long long> params,
                                     std::vector<unsigned long long> sigs, torch::Tensor momentum, size_t n_vec, double lr, double mu,
                                     double wd, bool nesterov, double scale, bool zero_grad, int rank, int world, int max_blocks) {
    sharded_sgd("sharded_sgd", bf16, grads, params, sigs, momentum, c10::nullopt, {lr}, {wd}, nullptr, n_vec, mu, nesterov, scale,
                zero_grad, rank, world, max_blocks);
  }, py::arg("bf16"), py::arg("grads"), py::arg("params"), py::arg("sigs"), py::arg("momentum"), py::arg("n_vec"), py::arg("lr"),
     py::arg("mu"), py::arg("weight_decay"), py::arg("nesterov"), py::arg("scale"), py::arg("zero_grad"), py::arg("rank"),
     py::arg("world"), py::arg("max_blocks") = 0);
  m.def("sharded_sgd_grouped", [sharded_sgd](bool bf16, std::vector<unsigned long long> grads, std::vector<unsigned long long> params,
                                             std::vector<unsigned long long> sigs, torch::Tensor momentum, torch::Tensor group_map,
                                             size_t n_vec, std::vector<double> lrs, std::vector<double> weight_decays, double mu,
                                             bool nesterov, double scale, bool zero_grad, int rank, int world, int max_blocks) {
    sharded_sgd("sharded_sgd_grouped", bf16, grads, params, sigs, momentum, group_map, lrs, weight_decays, nullptr, n_vec, mu, nesterov,
                scale, zero_grad, rank, world, max_blocks);
  }, py::arg("bf16"), py::arg("grads"), py::arg("params"), py::arg("sigs"), py::arg("momentum"), py::arg("group_map"),
     py::arg("n_vec"), py::arg("lrs"), py::arg("weight_decays"), py::arg("mu"), py::arg("nesterov"), py::arg("scale"),
     py::arg("zero_grad"), py::arg("rank"), py::arg("world"), py::arg("max_blocks") = 0);
  m.def("sharded_sgd_cap", [sharded_sgd](bool bf16, std::vector<unsigned long long> grads, std::vector<unsigned long long> params,
                                         std::vector<unsigned long long> sigs, torch::Tensor momentum,
                                         c10::optional<torch::Tensor> group_map, torch::Tensor block, size_t n_vec, double mu,
                                         bool nesterov, double scale, bool zero_grad, int rank, int world, int max_blocks) {
    sharded_sgd("sharded_sgd_cap", bf16, grads, params, sigs, momentum, group_map, {}, {}, &block, n_vec, mu, nesterov, scale, zero_grad,
                rank, world, max_blocks);
  }, py::arg("bf16"), py::arg("grads"), py::arg("params"), py::arg("sigs"), py::arg("momentum"), py::arg("group_map"),
     py::arg("block"), py::arg("n_vec"), py::arg("mu"), py::arg("nesterov"), py::arg("scale"), py::arg("zero_grad"),
     py::arg("rank"), py::arg("world"), py::arg("max_blocks") = 0);
  // The sharded step of one bucket with AdamW (csrc/sharded_sgd.cu, the AdamW instances): as sharded_sgd, with this rank's
  // exp_avg / exp_avg_sq shards in place of the momentum shard; group_map, decays / step_sizes and block as adamw_flat's.
  auto sharded_adamw = [](const char* what, bool bf16, const std::vector<unsigned long long>& grads,
                          const std::vector<unsigned long long>& params, const std::vector<unsigned long long>& sigs,
                          torch::Tensor& exp_avg, torch::Tensor& exp_avg_sq, const c10::optional<torch::Tensor>& group_map,
                          const std::vector<double>* scalars, const std::vector<double>& decays, const std::vector<double>& step_sizes,
                          const torch::Tensor* block, size_t n_vec, double scale, bool zero_grad, int rank, int world, int max_blocks) {
    const Peers pr = sharded_peers(what, grads, params, nullptr, sigs, n_vec, bf16, rank, world);
    const b2::AdamwScalars sc = scalars != nullptr ? to_adamw(*scalars, what) : b2::AdamwScalars{};
    check_flats({&exp_avg, &exp_avg_sq}, pr.shard, true, "exp_avg and exp_avg_sq (this rank's slice)", what);
    c10::cuda::CUDAGuard guard(exp_avg.device());
    if (block != nullptr) {
      ck_cuda(b2_sharded_adamw_cap_launch(bf16 ? 1 : 0, &pr.grads, &pr.params, &pr.sigs, exp_avg.data_ptr<float>(),
                                          exp_avg_sq.data_ptr<float>(), flat_map(group_map, pr.shard / 4, what),
                                          flat_block(*block, exp_avg, what), n_vec, (float)scale, zero_grad ? 1 : 0, rank, world,
                                          max_blocks, cur_stream()),
              what);
    } else if (group_map.has_value()) {
      b2::AdamwGroups gs;
      memset(&gs, 0, sizeof(gs));
      const int n_groups = check_groups(*group_map, pr.shard / 4, decays, step_sizes, gs.decay, gs.step_size, what);
      ck_cuda(b2_sharded_adamw_grouped_launch(bf16 ? 1 : 0, &pr.grads, &pr.params, &pr.sigs, exp_avg.data_ptr<float>(),
                                              exp_avg_sq.data_ptr<float>(), group_map->data_ptr<uint8_t>(), &sc, &gs, n_groups, n_vec,
                                              (float)scale, zero_grad ? 1 : 0, rank, world, max_blocks, cur_stream()),
              what);
    } else {
      ck_cuda(b2_sharded_adamw_launch(bf16 ? 1 : 0, &pr.grads, &pr.params, &pr.sigs, exp_avg.data_ptr<float>(),
                                      exp_avg_sq.data_ptr<float>(), n_vec, &sc, (float)scale, zero_grad ? 1 : 0, rank, world,
                                      max_blocks, cur_stream()),
              what);
    }
  };
  m.def("sharded_adamw", [sharded_adamw](bool bf16, std::vector<unsigned long long> grads, std::vector<unsigned long long> params,
                                         std::vector<unsigned long long> sigs, torch::Tensor exp_avg, torch::Tensor exp_avg_sq,
                                         size_t n_vec, std::vector<double> scalars, double scale, bool zero_grad, int rank, int world,
                                         int max_blocks) {
    sharded_adamw("sharded_adamw", bf16, grads, params, sigs, exp_avg, exp_avg_sq, c10::nullopt, &scalars, {}, {}, nullptr, n_vec,
                  scale, zero_grad, rank, world, max_blocks);
  }, py::arg("bf16"), py::arg("grads"), py::arg("params"), py::arg("sigs"), py::arg("exp_avg"), py::arg("exp_avg_sq"),
     py::arg("n_vec"), py::arg("scalars"), py::arg("scale"), py::arg("zero_grad"), py::arg("rank"), py::arg("world"),
     py::arg("max_blocks") = 0);
  m.def("sharded_adamw_grouped", [sharded_adamw](bool bf16, std::vector<unsigned long long> grads,
                                                 std::vector<unsigned long long> params, std::vector<unsigned long long> sigs,
                                                 torch::Tensor exp_avg, torch::Tensor exp_avg_sq, torch::Tensor group_map, size_t n_vec,
                                                 std::vector<double> scalars, std::vector<double> decays,
                                                 std::vector<double> step_sizes, double scale, bool zero_grad, int rank, int world,
                                                 int max_blocks) {
    sharded_adamw("sharded_adamw_grouped", bf16, grads, params, sigs, exp_avg, exp_avg_sq, group_map, &scalars, decays, step_sizes,
                  nullptr, n_vec, scale, zero_grad, rank, world, max_blocks);
  }, py::arg("bf16"), py::arg("grads"), py::arg("params"), py::arg("sigs"), py::arg("exp_avg"), py::arg("exp_avg_sq"),
     py::arg("group_map"), py::arg("n_vec"), py::arg("scalars"), py::arg("decays"), py::arg("step_sizes"), py::arg("scale"),
     py::arg("zero_grad"), py::arg("rank"), py::arg("world"), py::arg("max_blocks") = 0);
  m.def("sharded_adamw_cap", [sharded_adamw](bool bf16, std::vector<unsigned long long> grads, std::vector<unsigned long long> params,
                                             std::vector<unsigned long long> sigs, torch::Tensor exp_avg, torch::Tensor exp_avg_sq,
                                             c10::optional<torch::Tensor> group_map, torch::Tensor block, size_t n_vec, double scale,
                                             bool zero_grad, int rank, int world, int max_blocks) {
    sharded_adamw("sharded_adamw_cap", bf16, grads, params, sigs, exp_avg, exp_avg_sq, group_map, nullptr, {}, {}, &block, n_vec, scale,
                  zero_grad, rank, world, max_blocks);
  }, py::arg("bf16"), py::arg("grads"), py::arg("params"), py::arg("sigs"), py::arg("exp_avg"), py::arg("exp_avg_sq"),
     py::arg("group_map"), py::arg("block"), py::arg("n_vec"), py::arg("scale"), py::arg("zero_grad"), py::arg("rank"),
     py::arg("world"), py::arg("max_blocks") = 0);

  // ------------------------------------------------------------------ fused ConvNet step
  m.def("convnet_npar", [] { return b2_convnet_npar(); });
  m.def("convnet_smem_bytes", [] { return b2_convnet_smem_bytes(); });
  m.def("convnet_step", [](torch::Tensor params, c10::optional<torch::Tensor> grads, torch::Tensor x, torch::Tensor target,
                           c10::optional<torch::Tensor> loss_acc, c10::optional<torch::Tensor> out_logp,
                           c10::optional<torch::Tensor> mask_out, c10::optional<torch::Tensor> step, uint64_t seed,
                           int64_t sample_base, bool training, double inv_bsz, double p_drop, int max_ctas, int64_t grad_stride, int cluster,
                           c10::optional<torch::Tensor> aux, py::none, c10::optional<torch::Tensor> det_partials,
                           c10::optional<torch::Tensor> factors, bool input_ready) {
    // The kernels read params, x and aux with bulk copies and 16-byte vector loads, and write grads, det_partials and
    // factors with 16-byte vector stores / red.add.v4: a buffer that is not 16-byte aligned would fault on the device.
    auto check_aligned16 = [](const torch::Tensor& t, const char* what) {
      TORCH_CHECK(((uintptr_t)t.data_ptr() & 15u) == 0, "convnet_step: ", what, " must be 16-byte aligned");
    };
    check_cuda_contig(params, "params"); check_cuda_contig(x, "x"); check_cuda_contig(target, "target");
    TORCH_CHECK(params.scalar_type() == torch::kFloat32 && params.numel() >= b2_convnet_npar(), "params: flat fp32 [21848]");
    TORCH_CHECK(target.scalar_type() == torch::kInt64, "target: int64");
    check_aligned16(params, "params"); check_aligned16(x, "x");
    const bool u8 = x.scalar_type() == torch::kUInt8;
    TORCH_CHECK(u8 || x.scalar_type() == torch::kFloat32, "x: float32 (normalised) or uint8 (raw)");
    const int B = (int)target.numel();
    TORCH_CHECK(x.numel() == (int64_t)B * 784, "x must be [B,1,28,28]");
    float* g = nullptr;
    if (grads.has_value()) {
      check_cuda_contig(*grads, "grads"); check_aligned16(*grads, "grads");
      TORCH_CHECK(grad_stride >= 0 && grad_stride % 4 == 0, "convnet_step: grad_stride must be a non-negative multiple of 4 "
                  "(the second bucket is written with 16-byte vectors), got ", grad_stride);
      TORCH_CHECK(grads->scalar_type() == torch::kFloat32 && grads->numel() >= b2_convnet_npar() + grad_stride);
      g = grads->data_ptr<float>();
    }
    float* la = loss_acc.has_value() ? loss_acc->data_ptr<float>() : nullptr;
    float* lp = nullptr;
    if (out_logp.has_value()) { TORCH_CHECK(out_logp->numel() == (int64_t)B * 10 && out_logp->scalar_type() == torch::kFloat32); lp = out_logp->data_ptr<float>(); }
    float* mo = nullptr;
    if (mask_out.has_value()) { TORCH_CHECK(mask_out->numel() == (int64_t)B * 70 && mask_out->scalar_type() == torch::kFloat32); mo = mask_out->data_ptr<float>(); }
    const unsigned long long* st = step.has_value() ? reinterpret_cast<const unsigned long long*>(step->data_ptr()) : nullptr;
    c10::cuda::CUDAGuard guard(params.device());
    const float* ax = nullptr;
    if (aux.has_value()) {
      TORCH_CHECK(aux->is_cuda() && aux->scalar_type() == torch::kFloat32 && aux->numel() >= 13000);
      check_aligned16(*aux, "aux");
      ax = aux->data_ptr<float>();
    }
    float* dp = nullptr;
    if (det_partials.has_value()) {
      const int ctas = cluster > 1 ? B * cluster : (max_ctas > 0 ? std::min(B, max_ctas) : B);   // CTAs of the step grid
      TORCH_CHECK(det_partials->is_cuda() && det_partials->scalar_type() == torch::kFloat32 &&
                  det_partials->numel() >= (int64_t)std::max(1, ctas) * 21888, "det_partials: [ctas, 21888] fp32");
      check_aligned16(*det_partials, "det_partials");
      dp = det_partials->data_ptr<float>();
    }
    float* fp = nullptr;
    if (factors.has_value()) {
      // per-sample fc1 factors instead of fc1.weight in the slots (summed by reduce_sgd); one CTA per sample group only
      TORCH_CHECK(dp != nullptr && cluster <= 1, "factors need det_partials and cluster 1");
      TORCH_CHECK(factors->is_cuda() && factors->scalar_type() == torch::kFloat32 && factors->numel() >= (int64_t)std::max(1, B) * 384,
                  "factors: [B, 384] fp32");
      check_aligned16(*factors, "factors");
      fp = factors->data_ptr<float>();
    }
    if (cluster > 1) {
      TORCH_CHECK(cluster == 2 || cluster == 4 || cluster == 8, "cluster must be 1, 2, 4 or 8");
      ck_cuda(b2_convnet_cluster_launch(params.data_ptr<float>(), g, x.data_ptr(), u8, reinterpret_cast<const long long*>(target.data_ptr<int64_t>()),
                                        la, lp, mo, st, seed, sample_base, B, training, g != nullptr, (float)inv_bsz, (float)p_drop,
                                        cluster, max_ctas, grad_stride, ax, dp, cur_stream()), "convnet_cluster launch");
      return;
    }
    // input_ready: x and target were not written by the kernel right before this launch, so the step kernel may read them
    // before its griddepcontrol.wait (Args::input_ready)
    ck_cuda(b2_convnet_step_launch(params.data_ptr<float>(), g, x.data_ptr(), u8, reinterpret_cast<const long long*>(target.data_ptr<int64_t>()),
                                   la, lp, mo, st, seed, sample_base, B, training, g != nullptr, (float)inv_bsz, (float)p_drop,
                                   max_ctas, grad_stride, ax, dp, fp, input_ready ? 1 : 0, cur_stream()),
            "convnet_step launch");
  }, "Fused forward (+ loss and backward when grads is given) of the ConvNet on one CTA or one 2/4/8-CTA cluster per "
     "sample.  params, x, grads, aux, det_partials and factors must be 16-byte aligned (refused otherwise), and "
     "grad_stride a multiple of 4.",
     py::arg("params"), py::arg("grads"), py::arg("x"), py::arg("target"), py::arg("loss_acc"), py::arg("out_logp"),
     py::arg("mask_out"), py::arg("step"), py::arg("seed"), py::arg("sample_base"), py::arg("training"), py::arg("inv_bsz"),
     py::arg("p_drop") = 0.5, py::arg("max_ctas") = 0, py::arg("grad_stride") = 0, py::arg("cluster") = 1, py::arg("aux") = py::none(),
     // "reserved": an unused slot that takes only None, so calls passing det_partials, factors and input_ready by position
     // keep their meaning
     py::arg("reserved") = py::none(), py::arg("det_partials") = py::none(), py::arg("factors") = py::none(),
     py::arg("input_ready") = false);
  // ------------------------------------------------------------------ forward-only evaluation (csrc/convnet_eval.cu)
  m.def("convnet_eval_slot_words", [](int dev) {
    const int n = b2_convnet_eval_max_ctas(dev);
    TORCH_CHECK(n > 0, "convnet_eval: cannot configure the kernel on device ", dev);
    return 2 + 2 * n;
  }, "int32 words of the slot buffer convnet_eval needs on device `dev` (ticket + one (loss, #correct) pair per CTA)");
  m.def("convnet_eval_samples_per_cta", [] { return b2_convnet_eval_samples_per_cta(); });
  m.def("convnet_eval", [](torch::Tensor params, torch::Tensor x, torch::Tensor target, torch::Tensor result, torch::Tensor slots,
                           double mean, double std, c10::optional<torch::Tensor> out_logp) {
    check_cuda_contig(params, "params"); check_cuda_contig(x, "x"); check_cuda_contig(target, "target");
    check_cuda_contig(result, "result"); check_cuda_contig(slots, "slots");
    TORCH_CHECK(params.scalar_type() == torch::kFloat32 && params.numel() >= b2_convnet_npar(), "params: flat fp32 [21848]");
    TORCH_CHECK(target.scalar_type() == torch::kInt64, "target: int64");
    const bool u8 = x.scalar_type() == torch::kUInt8;
    TORCH_CHECK(u8 || x.scalar_type() == torch::kFloat32, "x: float32 (normalised) or uint8 (raw)");
    const int64_t N = target.numel();
    TORCH_CHECK(x.numel() == N * 784, "x must be [N,28,28] (uint8) or [N,1,28,28] (float32)");
    TORCH_CHECK(result.scalar_type() == torch::kFloat64 && result.numel() >= 3, "result: CUDA float64 [3]");
    TORCH_CHECK(slots.scalar_type() == torch::kInt32, "slots: CUDA int32");
    TORCH_CHECK(std > 0.0, "std must be positive");
    const auto dev = params.device();
    TORCH_CHECK(x.device() == dev && target.device() == dev && result.device() == dev && slots.device() == dev,
                "params, x, target, result and slots must be on one device");
    // the weights and each group's images arrive by 1-D bulk copies: 16-byte aligned sources
    TORCH_CHECK(((uintptr_t)params.data_ptr() | (uintptr_t)x.data_ptr()) % 16 == 0, "params and x must be 16-byte aligned");
    float* lp = nullptr;
    if (out_logp.has_value()) {
      check_cuda_contig(*out_logp, "out_logp");
      TORCH_CHECK(out_logp->numel() == N * 10 && out_logp->scalar_type() == torch::kFloat32 && out_logp->device() == dev,
                  "out_logp: CUDA float32 [N,10]");
      lp = out_logp->data_ptr<float>();
    }
    c10::cuda::CUDAGuard guard(dev);
    const int max_ctas = b2_convnet_eval_max_ctas(dev.index());
    TORCH_CHECK(max_ctas > 0, "convnet_eval: cannot configure the kernel on ", dev);
    TORCH_CHECK(slots.numel() >= 2 + 2 * (int64_t)max_ctas, "slots: int32 [convnet_eval_slot_words(device)], zero-initialised");
    ck_cuda(b2_convnet_eval_launch(params.data_ptr<float>(), x.data_ptr(), u8 ? 1 : 0,
                                   reinterpret_cast<const long long*>(target.data_ptr<int64_t>()), result.data_ptr<double>(),
                                   slots.data_ptr<int>(), lp, N, (float)mean, (float)std, dev.index(), cur_stream()),
            "convnet_eval launch");
  }, py::arg("params"), py::arg("x"), py::arg("target"), py::arg("result"), py::arg("slots"), py::arg("mean"), py::arg("std"),
     py::arg("out_logp") = py::none());
  m.def("reduce_sgd", [](torch::Tensor slots, int n_slots, torch::Tensor factors, int n_samples, torch::Tensor params,
                         torch::Tensor momentum, c10::optional<torch::Tensor> step, c10::optional<torch::Tensor> done_counter,
                         double lr, double mu, c10::optional<torch::Tensor> aux, c10::optional<torch::Tensor> loss_acc,
                         c10::optional<torch::Tensor> grads, int64_t grad_stride, py::object lr_schedule, double weight_decay,
                         bool nesterov, py::object max_grad_norm, c10::optional<torch::Tensor> clip_workspace,
                         c10::optional<torch::Tensor> grad_norm_out, int n_cta) {
    // one-GPU optimizer step from convnet_step(..., det_partials=slots, factors=factors): the local gradient is summed from
    // the first n_slots slots and n_samples factor rows in a fixed order, then SGD is applied to it.  The gradient bucket is
    // not read; given `grads`, its other-parity half is re-zeroed like allreduce_sgd does, so a bucket step may follow.
    // n_cta: the kernel's grid; 0 is min(SMs, RED_UNITS), the grid every trainer uses.  A smaller grid runs several reduction
    // units per CTA, as on a card with fewer SMs.  A CTA past the last unit never reaches its first unit's check-in on
    // done_counter, so the step counter would never advance: grids above RED_UNITS are refused.
    check_cuda_contig(slots, "slots"); check_cuda_contig(factors, "factors");
    check_cuda_contig(params, "params"); check_cuda_contig(momentum, "momentum");
    TORCH_CHECK(slots.scalar_type() == torch::kFloat32 && slots.numel() >= (int64_t)n_slots * 21888, "slots: [n_slots, 21888] fp32");
    TORCH_CHECK(factors.scalar_type() == torch::kFloat32 && factors.numel() >= (int64_t)n_samples * 384, "factors: [n_samples, 384] fp32");
    TORCH_CHECK(params.scalar_type() == torch::kFloat32 && momentum.scalar_type() == torch::kFloat32 &&
                params.numel() >= b2_convnet_npar() && params.numel() == momentum.numel(), "fp32 flat buffers");
    unsigned long long* st = step.has_value() ? reinterpret_cast<unsigned long long*>(step->data_ptr()) : nullptr;
    unsigned int* dc = done_counter.has_value() ? reinterpret_cast<unsigned int*>(done_counter->data_ptr()) : nullptr;
    TORCH_CHECK(st == nullptr || dc != nullptr, "a step counter needs a done_counter scratch word");
    float* ax = nullptr;
    if (aux.has_value()) { TORCH_CHECK(aux->is_cuda() && aux->scalar_type() == torch::kFloat32 && aux->numel() >= 13000); ax = aux->data_ptr<float>(); }
    float* la = loss_acc.has_value() ? loss_acc->data_ptr<float>() : nullptr;
    float* g = nullptr;
    if (grads.has_value()) {
      check_cuda_contig(*grads, "grads");
      TORCH_CHECK(grads->scalar_type() == torch::kFloat32 && grad_stride >= 0 && grads->numel() >= b2_convnet_npar() + grad_stride,
                  "grads: fp32 [npar + grad_stride]");
      g = grads->data_ptr<float>();
    }
    const b2::LrSchedule sched = to_sched(lr_schedule);
    check_sgd_options(weight_decay, nesterov, mu, "reduce_sgd");
    TORCH_CHECK(n_cta >= 0 && n_cta <= b2_reduce_units(), "reduce_sgd: n_cta must be 0 (the default grid) or 1..",
                b2_reduce_units(), ", got ", n_cta);
    const float max_norm = check_max_grad_norm(max_grad_norm, "reduce_sgd");
    float* ws = clip_ws_ptr(max_norm, clip_workspace, params.numel(), "reduce_sgd");
    float* gn = grad_norm_ptr(grad_norm_out, "reduce_sgd");
    c10::cuda::CUDAGuard guard(params.device());
    ck_cuda(b2_reduce_sgd_launch(params.data_ptr<float>(), momentum.data_ptr<float>(), st, dc, (float)lr, (float)mu, ax, la, nullptr,
                                 slots.data_ptr<float>(), n_slots, factors.data_ptr<float>(), n_samples, g, grad_stride, &sched,
                                 (float)weight_decay, nesterov ? 1 : 0, max_norm, ws, gn, n_cta, cur_stream()),
            "reduce_sgd launch");
  }, py::arg("slots"), py::arg("n_slots"), py::arg("factors"), py::arg("n_samples"), py::arg("params"), py::arg("momentum"),
     py::arg("step"), py::arg("done_counter"), py::arg("lr"), py::arg("mu"), py::arg("aux") = py::none(), py::arg("loss_acc") = py::none(),
     py::arg("grads") = py::none(), py::arg("grad_stride") = 0, py::arg("lr_schedule") = py::none(),
     py::arg("weight_decay") = 0.0, py::arg("nesterov") = false, py::arg("max_grad_norm") = py::none(),
     py::arg("clip_workspace") = py::none(), py::arg("grad_norm_out") = py::none(), py::arg("n_cta") = 0);
  m.def("lr_schedule_eval", [](py::object schedule, double lr, torch::Tensor steps) {
    // the fp32 lr the optimizer kernels apply at each step-counter value of `steps`, computed by the same device function
    check_cuda_contig(steps, "steps");
    TORCH_CHECK(steps.scalar_type() == torch::kInt64, "steps: CUDA int64");
    const b2::LrSchedule sched = to_sched(schedule);
    auto out = torch::empty({steps.numel()}, steps.options().dtype(torch::kFloat32));
    c10::cuda::CUDAGuard guard(steps.device());
    ck_cuda(b2_lr_schedule_eval_launch(&sched, (float)lr, reinterpret_cast<const long long*>(steps.data_ptr<int64_t>()),
                                       out.data_ptr<float>(), steps.numel(), cur_stream()), "lr_schedule_eval launch");
    return out;
  }, py::arg("schedule"), py::arg("lr"), py::arg("steps"));
  m.def("set_phase_ts", [](c10::optional<torch::Tensor> ts) {
    // opt-in phase timestamps of later step / optimizer launches (bench/step_phases.py); None turns them off
    if (ts.has_value()) TORCH_CHECK(ts->is_cuda() && ts->scalar_type() == torch::kInt64 && ts->numel() >= 64 * 256 * 16, "ts: int64 [64*256*16]");
    b2_set_phase_ts(ts.has_value() ? reinterpret_cast<unsigned long long*>(ts->data_ptr()) : nullptr);
  }, py::arg("ts"));
  m.def("det_reduce", [](torch::Tensor partials, int n_slots, torch::Tensor grads, c10::optional<torch::Tensor> step, int64_t grad_stride,
                         c10::optional<torch::Tensor> loss_acc) {
    // deterministic mode: grads[(step & 1) * grad_stride ...] = sum over the first n_slots per-CTA slots, in slot order
    check_cuda_contig(partials, "partials"); check_cuda_contig(grads, "grads");
    TORCH_CHECK(partials.scalar_type() == torch::kFloat32 && grads.scalar_type() == torch::kFloat32 && partials.numel() >= (int64_t)n_slots * 21888);
    const unsigned long long* st = step.has_value() ? reinterpret_cast<const unsigned long long*>(step->data_ptr()) : nullptr;
    c10::cuda::CUDAGuard guard(grads.device());
    float* la = loss_acc.has_value() ? loss_acc->data_ptr<float>() : nullptr;
    ck_cuda(b2_det_reduce_launch(partials.data_ptr<float>(), n_slots, 21888, grads.data_ptr<float>(), st, grad_stride,
                                 (size_t)b2_convnet_npar(), la, cur_stream()), "det_reduce launch");
  }, py::arg("partials"), py::arg("n_slots"), py::arg("grads"), py::arg("step") = py::none(), py::arg("grad_stride") = 0,
     py::arg("loss_acc") = py::none());

  // ------------------------------------------------------------------ wgmma GEMM
  m.def("gemm_available", [] { return b2_gemm_available() != 0; });
  m.def("gemm_bf16", [](torch::Tensor a, torch::Tensor b, c10::optional<torch::Tensor> bias, bool relu, bool out_bf16,
                        c10::optional<torch::Tensor> out) {
    // C[M,N] = A[M,K] @ B[N,K]^T (+bias) (relu) ; A,B bf16 row-major (K contiguous).  `out`, if given, receives C in place
    // (a contiguous [M,N] tensor of the output dtype on A's device, 16-byte aligned), as the batched engine's fixed buffers do.
    check_cuda_contig(a, "a"); check_cuda_contig(b, "b");
    TORCH_CHECK(a.scalar_type() == torch::kBFloat16 && b.scalar_type() == torch::kBFloat16, "bf16 operands");
    TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && a.size(1) == b.size(1), "A[M,K], B[N,K]");
    const int M = (int)a.size(0), K = (int)a.size(1), N = (int)b.size(0);
    TORCH_CHECK(K % 8 == 0, "K must be a multiple of 8 (16-byte rows for TMA)");
    const float* bp = nullptr;
    if (bias.has_value()) { TORCH_CHECK(bias->is_cuda() && bias->scalar_type() == torch::kFloat32 && bias->numel() == N); bp = bias->data_ptr<float>(); }
    const auto out_dtype = out_bf16 ? torch::kBFloat16 : torch::kFloat32;
    torch::Tensor c;
    if (out.has_value()) {
      c = *out;
      TORCH_CHECK(c.is_cuda() && c.device() == a.device(), "gemm_bf16: out must be on the operands' device");
      TORCH_CHECK(c.scalar_type() == out_dtype, "gemm_bf16: out must be ", out_bf16 ? "bf16" : "fp32");
      TORCH_CHECK(c.dim() == 2 && c.size(0) == M && c.size(1) == N, "gemm_bf16: out must have shape [M, N]");
      TORCH_CHECK(c.is_contiguous(), "gemm_bf16: out must be contiguous");
      TORCH_CHECK((reinterpret_cast<uintptr_t>(c.data_ptr()) & 15) == 0, "gemm_bf16: out must be 16-byte aligned");
    } else {
      c = torch::empty({M, N}, a.options().dtype(out_dtype));
    }
    c10::cuda::CUDAGuard guard(a.device());
    int rc = b2_gemm_bf16_launch(a.data_ptr(), b.data_ptr(), c.data_ptr(), bp, M, N, K, relu, out_bf16, cur_stream());
    if (rc != 0) throw std::runtime_error(std::string("gemm_bf16: ") + b2_gemm_last_error());
    return c;
  }, py::arg("a"), py::arg("b"), py::arg("bias") = py::none(), py::arg("relu") = false, py::arg("out_bf16") = true,
     py::arg("out") = py::none());

  // ------------------------------------------------------------------ batched tensor-core engine (csrc/convnet_batched.cu)
  // bufs: [P1, P2, H, DH, dP2, DC, W2K, W2R, W3K, W3T, A1, A2, Hrelu, DLOG, G1, B3P] (see ops/convnet_batched.py)
  auto bt_bufs = [](const std::vector<torch::Tensor>& v, int64_t B) {
    TORCH_CHECK(v.size() == 16, "bufs: 16 tensors");
    const int64_t need[16] = {B * 2304, B * 320, B * 64, B * 64, B * 320, B * 2048, 32 * 448, 400 * 64, 64 * 320, 320 * 64,
                              B * 1440, B * 320, B * 64, B * 16, B * 1440, 64};
    for (int i = 0; i < 16; ++i) {
      TORCH_CHECK(v[i].is_cuda() && v[i].is_contiguous() && v[i].numel() >= need[i], "bufs[", i, "] too small / not CUDA");
      const auto want = i < 10 ? torch::kBFloat16 : (i < 12 ? torch::kUInt8 : torch::kFloat32);
      TORCH_CHECK(v[i].scalar_type() == want, "bufs[", i, "] dtype");
      TORCH_CHECK(((uintptr_t)v[i].data_ptr() & 127) == 0, "bufs[", i, "] must be 128-byte aligned");
    }
    BtBuffers b;
    b.P1 = v[0].data_ptr(); b.P2 = v[1].data_ptr(); b.H = v[2].data_ptr(); b.DH = v[3].data_ptr(); b.dP2 = v[4].data_ptr();
    b.DC = v[5].data_ptr(); b.W2K = v[6].data_ptr(); b.W2R = v[7].data_ptr(); b.W3K = v[8].data_ptr(); b.W3T = v[9].data_ptr();
    b.A1 = v[10].data_ptr<uint8_t>(); b.A2 = v[11].data_ptr<uint8_t>();
    b.Hrelu = v[12].data_ptr<float>(); b.DLOG = v[13].data_ptr<float>(); b.G1 = v[14].data_ptr<float>(); b.B3P = v[15].data_ptr<float>();
    return b;
  };
  m.def("bt_pack_weights", [bt_bufs](torch::Tensor params, std::vector<torch::Tensor> bufs) {
    check_cuda_contig(params, "params");
    TORCH_CHECK(params.scalar_type() == torch::kFloat32 && params.numel() >= b2_convnet_npar());
    BtBuffers b = bt_bufs(bufs, 0);
    c10::cuda::CUDAGuard guard(params.device());
    ck_cuda(b2_bt_pack_weights(params.data_ptr<float>(), &b, cur_stream()), "bt_pack_weights launch");
  });
  m.def("bt_step", [bt_bufs](torch::Tensor params, c10::optional<torch::Tensor> grads, torch::Tensor x, torch::Tensor target,
                             std::vector<torch::Tensor> bufs, c10::optional<torch::Tensor> loss_acc,
                             c10::optional<torch::Tensor> out_logp, c10::optional<torch::Tensor> step, uint64_t seed,
                             int64_t sample_base, bool training, double inv_bsz, double p_drop, int stage_mask) {
    check_cuda_contig(params, "params"); check_cuda_contig(x, "x"); check_cuda_contig(target, "target");
    TORCH_CHECK(params.scalar_type() == torch::kFloat32 && params.numel() >= b2_convnet_npar(), "params: flat fp32 [21848]");
    TORCH_CHECK(target.scalar_type() == torch::kInt64, "target: int64");
    const bool u8 = x.scalar_type() == torch::kUInt8;
    TORCH_CHECK(u8 || x.scalar_type() == torch::kFloat32, "x: float32 (normalised) or uint8 (raw)");
    const int B = (int)target.numel();
    TORCH_CHECK(x.numel() == (int64_t)B * 784, "x must be [B,1,28,28]");
    float* g = nullptr;
    if (grads.has_value()) { check_cuda_contig(*grads, "grads"); TORCH_CHECK(grads->scalar_type() == torch::kFloat32 && grads->numel() >= b2_convnet_npar()); g = grads->data_ptr<float>(); }
    float* la = loss_acc.has_value() ? loss_acc->data_ptr<float>() : nullptr;
    float* lp = nullptr;
    if (out_logp.has_value()) { TORCH_CHECK(out_logp->numel() == (int64_t)B * 10 && out_logp->scalar_type() == torch::kFloat32); lp = out_logp->data_ptr<float>(); }
    const unsigned long long* st = step.has_value() ? reinterpret_cast<const unsigned long long*>(step->data_ptr()) : nullptr;
    BtBuffers b = bt_bufs(bufs, B);
    c10::cuda::CUDAGuard guard(params.device());
    int rc = b2_bt_step_launch(params.data_ptr<float>(), g, x.data_ptr(), u8, reinterpret_cast<const long long*>(target.data_ptr<int64_t>()),
                               &b, la, lp, st, seed, sample_base, B, training, g != nullptr, (float)inv_bsz, (float)p_drop,
                               stage_mask, cur_stream());
    if (rc != 0) throw std::runtime_error(std::string("bt_step: ") + b2_bt_last_error());
  }, py::arg("params"), py::arg("grads"), py::arg("x"), py::arg("target"), py::arg("bufs"), py::arg("loss_acc"),
     py::arg("out_logp"), py::arg("step"), py::arg("seed"), py::arg("sample_base"), py::arg("training"), py::arg("inv_bsz"),
     py::arg("p_drop") = 0.5, py::arg("stage_mask") = 255);

  // ------------------------------------------------------------------ tensor-core layout probes (tests/test_gpu_tc_probe.py)
  m.def("tma_probe", [](torch::Tensor tensor, std::vector<unsigned long long> dims, std::vector<unsigned long long> strides_bytes,
                        std::vector<unsigned int> box, int swizzle, std::vector<int> coords) {
    // one TMA box load of a uint16 tensor map -> the raw shared-memory image (uint8)
    check_cuda_contig(tensor, "tensor");
    const int rank = (int)dims.size();
    TORCH_CHECK(rank >= 2 && rank <= 5 && (int)box.size() == rank && (int)coords.size() == rank && (int)strides_bytes.size() == rank - 1);
    size_t bytes = 2;
    for (auto b : box) bytes *= b;
    coords.resize(5, 0);
    auto out = torch::zeros({(int64_t)bytes}, tensor.options().dtype(torch::kUInt8));
    c10::cuda::CUDAGuard guard(tensor.device());
    int rc = b2_tma_probe(tensor.data_ptr(), rank, dims.data(), strides_bytes.data(), box.data(), swizzle, coords.data(),
                          (unsigned int)bytes, out.data_ptr<uint8_t>(), cur_stream());
    if (rc != 0) throw std::runtime_error(std::string("tma_probe: ") + b2_probe_last_error());
    return out;
  }, py::arg("tensor"), py::arg("dims"), py::arg("strides_bytes"), py::arg("box"), py::arg("swizzle"), py::arg("coords"));
  m.def("wgmma_probe", [](torch::Tensor a_img, torch::Tensor b_img, bool a_mn, std::vector<unsigned long long> ops, int n) {
    // ops: flat list of (adesc, bdesc, accumulate) triples of one warpgroup; returns D[64, n] fp32
    check_cuda_contig(a_img, "a_img"); check_cuda_contig(b_img, "b_img");
    TORCH_CHECK(a_img.scalar_type() == torch::kUInt8 && b_img.scalar_type() == torch::kUInt8 && ops.size() % 3 == 0);
    auto dump = torch::zeros({64, n}, a_img.options().dtype(torch::kFloat32));
    c10::cuda::CUDAGuard guard(a_img.device());
    int rc = b2_wgmma_probe(a_img.data_ptr<uint8_t>(), (unsigned int)a_img.numel(), b_img.data_ptr<uint8_t>(), (unsigned int)b_img.numel(),
                            a_mn ? 1 : 0, ops.data(), (int)(ops.size() / 3), n, dump.data_ptr<float>(), cur_stream());
    if (rc != 0) throw std::runtime_error(std::string("wgmma_probe: ") + b2_probe_last_error());
    return dump;
  }, py::arg("a_img"), py::arg("b_img"), py::arg("a_mn"), py::arg("ops"), py::arg("n"));

  // ------------------------------------------------------------------ native step executor
  py::class_<ExecutorPy>(m, "StepExecutor")
      .def(py::init<LoaderPy&, torch::Tensor, torch::Tensor, torch::Tensor, std::vector<unsigned long long>,
                    std::vector<unsigned long long>, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, bool, bool,
                    int, int, uint64_t, int64_t, int64_t, double, double, double, int, int, torch::Tensor,
                    std::vector<unsigned long long>, torch::Tensor, bool, c10::optional<torch::Tensor>,
                    c10::optional<torch::Tensor>, py::object, double, bool, py::object, c10::optional<torch::Tensor>,
                    c10::optional<torch::Tensor>>(),
           py::arg("loader"), py::arg("params"), py::arg("momentum"), py::arg("grads"), py::arg("grad_ptrs"),
           py::arg("sig_ptrs"), py::arg("step"), py::arg("done_counter"), py::arg("loss_acc"), py::arg("in_dev"),
           py::arg("raw_u8"), py::arg("training"), py::arg("rank"), py::arg("world"), py::arg("seed"),
           py::arg("sample_base"), py::arg("grad_stride"), py::arg("lr"), py::arg("mu"), py::arg("p_drop"),
           py::arg("max_in_flight") = 3, py::arg("cluster") = 1, py::arg("aux") = torch::Tensor(),
           py::arg("inbox") = std::vector<unsigned long long>(), py::arg("loss_hist") = torch::Tensor(),
           py::arg("wire_bf16") = false, py::arg("grad_slots") = py::none(),
           py::arg("factors") = py::none(), py::arg("lr_schedule") = py::none(), py::arg("weight_decay") = 0.0,
           py::arg("nesterov") = false, py::arg("max_grad_norm") = py::none(), py::arg("clip_workspace") = py::none(),
           py::arg("grad_norm_out") = py::none(), py::keep_alive<1, 2>())
      .def("chunking", [](ExecutorPy&) { return false; })      // read by bench.py: every step is issued on its own
      .def("flag_mode", [](ExecutorPy&) { return false; })     // read by bench.py: the streams are ordered by events
      .def("stats", [](ExecutorPy& e) {
        const auto& s = e.impl->stats();
        py::dict d;
        d["next_us"] = s.next_ns / 1e3; d["retire_us"] = s.retire_ns / 1e3; d["total_us"] = s.total_ns / 1e3;
        d["steps"] = s.steps;
        return d;
      })
      .def("reset_stats", [](ExecutorPy& e) { e.impl->reset_stats(); })
      .def("run", &ExecutorPy::run, py::arg("max_steps") = -1)
      .def("drain", [](ExecutorPy& e) { py::gil_scoped_release nogil; e.impl->drain(); })
      .def("last_loss_cumulative", [](ExecutorPy& e) { return e.impl->last_loss_cumulative(); });

  // ------------------------------------------------------------------ native loader
  py::class_<LoaderPy>(m, "NativeLoader")
      .def(py::init<torch::Tensor, torch::Tensor, torch::Tensor, int64_t, int, bool, bool, bool, double, double, uint64_t, bool>(),
           py::arg("images"), py::arg("labels"), py::arg("index"), py::arg("batch"), py::arg("n_buffers") = 4,
           py::arg("shuffle") = true, py::arg("drop_last") = false, py::arg("raw_u8") = false, py::arg("mean") = 0.1307,
           py::arg("std") = 0.3081, py::arg("seed") = 1234, py::arg("pin") = false)
      .def("num_batches", [](LoaderPy& l) { return l.impl->num_batches(); })
      .def("start_epoch", [](LoaderPy& l, int64_t e) { py::gil_scoped_release nogil; l.impl->start_epoch(e); })
      .def("next", &LoaderPy::next)
      .def("release", [](LoaderPy& l) { l.impl->release(); })
      .def("block_bytes", [](LoaderPy& l) { return l.impl->block_bytes(); })
      .def("stop", [](LoaderPy& l) { py::gil_scoped_release nogil; l.impl->stop(); });
}
