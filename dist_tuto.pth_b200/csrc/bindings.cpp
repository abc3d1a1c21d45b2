// Python bindings (pybind11 / torch extension) for the native runtime and the sm_90a kernels.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "executor.h"
#include "loader.h"

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
int b2_barrier_launch(const SignalPadsH* sig, int rank, int world, cudaStream_t stream);
int b2_allreduce_sgd_launch(const PeerPtrs* grads, const SignalPadsH* sig, float* params, float* momentum,
                            unsigned long long* step, size_t n_elems, float lr, float mu, float scale, int rank,
                            int world, int zero_grads, long long grad_stride, unsigned int* done_counter, float* aux,
                            const PeerPtrs* inbox, const float* loss_acc, float* loss_snapshot, int wire_bf16,
                            const b2::LrSchedule* sched, cudaStream_t stream);
int b2_lr_schedule_eval_launch(const b2::LrSchedule* sched, float base, const long long* steps, float* out, long long n,
                               cudaStream_t stream);
int b2_sgd_flat_launch(float* p, float* m, const float* g, size_t n, float lr, float mu, float wd, int zero_grad,
                       cudaStream_t stream);
size_t b2_convnet_smem_bytes();
int b2_convnet_npar();
int b2_convnet_step_launch(const float* params, float* grads, const void* x, int x_u8, const long long* target,
                           float* loss_acc, float* out_logp, float* mask_out, const unsigned long long* step,
                           unsigned long long seed, long long sample_base, int B, int training, int backward,
                           float inv_bsz, float p_drop, int max_ctas, long long grad_stride, const float* aux,
                           float* det_partials, float* factors, int input_ready, cudaStream_t stream);
int b2_reduce_sgd_launch(float* params, float* momentum, unsigned long long* step, unsigned int* done_counter, float lr, float mu,
                         float* aux, float* loss_acc, float* loss_snapshot, const float* slots, int n_slots, const float* factors,
                         int n_samples, float* grads, long long grad_stride, const b2::LrSchedule* sched, cudaStream_t stream);
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
             py::object lr_schedule)
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
  // (n_vec counts the output, world x the per-rank input).  The raw moves take any dtype and copy bytes.
  auto collective = [](const char* what, int op, int variant, bool bf16, const std::vector<unsigned long long>& bufs,
                       const std::vector<unsigned long long>& sigs, unsigned long long mc, const c10::optional<torch::Tensor>& src,
                       const c10::optional<torch::Tensor>& dst, size_t n_vec, double scale, int root, int rank, int world,
                       int max_blocks, const std::vector<unsigned long long>& inbox, size_t ll_cap) {
    check_world(rank, world, what);
    TORCH_CHECK(variant >= 0 && variant <= 3, what, ": variant must be 0 (one-shot), 1 (two-shot), 2 (NVLS) or 3 (LL), got ",
                variant);
    TORCH_CHECK((int)bufs.size() == world && (int)sigs.size() == world, what, ": one buffer and one signal pad per rank, got ",
                bufs.size(), " and ", sigs.size(), " for world ", world);
    TORCH_CHECK(variant == 3 ? (int)inbox.size() == world : inbox.empty() || (int)inbox.size() == world,
                what, ": one LL inbox per rank, got ", inbox.size(), " for world ", world);
    TORCH_CHECK((variant != 1 && variant != 2 && op != 5) || n_vec % (size_t)world == 0,
                what, ": two-shot, NVLS and all-gather split n_vec into world slices, so n_vec must be a multiple of world "
                "(pad the buffer), got n_vec ", n_vec, " for world ", world);
    TORCH_CHECK(root >= -1 && root < world, what, ": root must be -1 (every rank) or in [0, world), got ", root,
                " for world ", world);
    TORCH_CHECK(op == 0 || scale == 1.0, what, ": scale applies to SUM only, got ", scale, " for op ", op);
    TORCH_CHECK(variant != 2 || (op == 0 && root < 0), what, ": NVLS runs the SUM all-reduce only");
    TORCH_CHECK(variant != 3 || (op == 5 ? n_vec / world : n_vec) <= ll_cap, what, ": LL pushes ",
                op == 5 ? n_vec / world : n_vec, " vectors per rank, more than the inbox holds (", ll_cap, ")");
    PeerPtrs b = to_ptrs(bufs); SignalPadsH s = to_sig(sigs);
    PeerPtrs ib = to_ptrs(inbox);
    const void* sp = nullptr; void* dp = nullptr; int sf = 0, df = 0;
    if (src.has_value()) { check_cuda_contig(*src, "src"); sp = src->data_ptr(); sf = src->scalar_type() == torch::kFloat32 && bf16; }
    if (dst.has_value()) { check_cuda_contig(*dst, "dst"); dp = dst->data_ptr(); df = dst->scalar_type() == torch::kFloat32 && bf16; }
    TORCH_CHECK(op == 0 || (sf == 0 && df == 0), what, ": a bf16 wire for fp32 tensors is for SUM only");
    ck_cuda(b2_allreduce_launch(variant, bf16, &b, &s, (void*)(uintptr_t)mc, sp, sf, dp, df, n_vec, (float)scale, rank,
                                world, max_blocks, inbox.empty() ? nullptr : &ib, ll_cap, op, root, cur_stream()), what);
  };
  m.def("allreduce", [collective](int variant, bool bf16, std::vector<unsigned long long> bufs, std::vector<unsigned long long> sigs,
                                  unsigned long long mc, c10::optional<torch::Tensor> src, c10::optional<torch::Tensor> dst,
                                  size_t n_vec, double scale, int rank, int world, int max_blocks, std::vector<unsigned long long> inbox,
                                  size_t ll_cap, int op, int root) {
    TORCH_CHECK(op >= 0 && op <= 3, "allreduce: op must be 0 (SUM), 1 (PRODUCT), 2 (MAX) or 3 (MIN), got ", op);
    collective("allreduce", op, variant, bf16, bufs, sigs, mc, src, dst, n_vec, scale, root, rank, world, max_blocks, inbox, ll_cap);
  }, py::arg("variant"), py::arg("bf16"), py::arg("bufs"), py::arg("sigs"), py::arg("mc"), py::arg("src"), py::arg("dst"),
     py::arg("n_vec"), py::arg("scale"), py::arg("rank"), py::arg("world"), py::arg("max_blocks") = 0,
     py::arg("inbox") = std::vector<unsigned long long>(), py::arg("ll_cap") = 0, py::arg("op") = 0, py::arg("root") = -1);
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
  m.def("barrier", [](std::vector<unsigned long long> sigs, int rank, int world) {
    check_world(rank, world, "barrier");
    TORCH_CHECK((int)sigs.size() == world, "barrier: one signal pad per rank, got ", sigs.size(), " for world ", world);
    SignalPadsH s = to_sig(sigs);
    ck_cuda(b2_barrier_launch(&s, rank, world, cur_stream()), "barrier launch");
  });
  m.def("allreduce_sgd", [](std::vector<unsigned long long> grads, std::vector<unsigned long long> sigs, torch::Tensor params,
                            torch::Tensor momentum, c10::optional<torch::Tensor> step, double lr, double mu, double scale,
                            int rank, int world, bool zero_grads, int64_t grad_stride, c10::optional<torch::Tensor> done_counter,
                            c10::optional<torch::Tensor> aux, std::vector<unsigned long long> inbox, bool wire_bf16,
                            py::object lr_schedule) {
    check_world(rank, world, "allreduce_sgd");
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
    c10::cuda::CUDAGuard guard(params.device());
    ck_cuda(b2_allreduce_sgd_launch(&g, &s, params.data_ptr<float>(), momentum.data_ptr<float>(), st, (size_t)params.numel(),
                                    (float)lr, (float)mu, (float)scale, rank, world, zero_grads, grad_stride, dc, ax,
                                    inbox.empty() ? nullptr : &ib, nullptr, nullptr, wire_bf16 ? 1 : 0, &sched, cur_stream()),
            "allreduce_sgd launch");
  }, py::arg("grads"), py::arg("sigs"), py::arg("params"), py::arg("momentum"), py::arg("step"), py::arg("lr"), py::arg("mu"),
     py::arg("scale"), py::arg("rank"), py::arg("world"), py::arg("zero_grads"), py::arg("grad_stride") = 0,
     py::arg("done_counter") = py::none(), py::arg("aux") = py::none(), py::arg("inbox") = std::vector<unsigned long long>(),
     py::arg("wire_bf16") = false, py::arg("lr_schedule") = py::none());
  m.def("sgd_flat", [](torch::Tensor p, torch::Tensor mom, torch::Tensor g, double lr, double mu, double wd, bool zero_grad) {
    check_cuda_contig(p, "p"); check_cuda_contig(mom, "m"); check_cuda_contig(g, "g");
    TORCH_CHECK(p.scalar_type() == torch::kFloat32 && g.scalar_type() == torch::kFloat32 && mom.scalar_type() == torch::kFloat32);
    TORCH_CHECK(p.numel() == g.numel() && p.numel() == mom.numel());
    TORCH_CHECK(((uintptr_t)p.data_ptr() | (uintptr_t)mom.data_ptr() | (uintptr_t)g.data_ptr()) % 16 == 0, "16-byte aligned buffers");
    ck_cuda(b2_sgd_flat_launch(p.data_ptr<float>(), mom.data_ptr<float>(), g.data_ptr<float>(), (size_t)p.numel(), (float)lr,
                               (float)mu, (float)wd, zero_grad, cur_stream()), "sgd_flat launch");
  });

  // ------------------------------------------------------------------ fused ConvNet step
  m.def("convnet_npar", [] { return b2_convnet_npar(); });
  m.def("convnet_smem_bytes", [] { return b2_convnet_smem_bytes(); });
  m.def("convnet_step", [](torch::Tensor params, c10::optional<torch::Tensor> grads, torch::Tensor x, torch::Tensor target,
                           c10::optional<torch::Tensor> loss_acc, c10::optional<torch::Tensor> out_logp,
                           c10::optional<torch::Tensor> mask_out, c10::optional<torch::Tensor> step, uint64_t seed,
                           int64_t sample_base, bool training, double inv_bsz, double p_drop, int max_ctas, int64_t grad_stride, int cluster,
                           c10::optional<torch::Tensor> aux, py::none, c10::optional<torch::Tensor> det_partials,
                           c10::optional<torch::Tensor> factors, bool input_ready) {
    check_cuda_contig(params, "params"); check_cuda_contig(x, "x"); check_cuda_contig(target, "target");
    TORCH_CHECK(params.scalar_type() == torch::kFloat32 && params.numel() >= b2_convnet_npar(), "params: flat fp32 [21848]");
    TORCH_CHECK(target.scalar_type() == torch::kInt64, "target: int64");
    const bool u8 = x.scalar_type() == torch::kUInt8;
    TORCH_CHECK(u8 || x.scalar_type() == torch::kFloat32, "x: float32 (normalised) or uint8 (raw)");
    const int B = (int)target.numel();
    TORCH_CHECK(x.numel() == (int64_t)B * 784, "x must be [B,1,28,28]");
    float* g = nullptr;
    if (grads.has_value()) { check_cuda_contig(*grads, "grads"); TORCH_CHECK(grads->scalar_type() == torch::kFloat32 && grads->numel() >= b2_convnet_npar() + grad_stride); g = grads->data_ptr<float>(); }
    float* la = loss_acc.has_value() ? loss_acc->data_ptr<float>() : nullptr;
    float* lp = nullptr;
    if (out_logp.has_value()) { TORCH_CHECK(out_logp->numel() == (int64_t)B * 10 && out_logp->scalar_type() == torch::kFloat32); lp = out_logp->data_ptr<float>(); }
    float* mo = nullptr;
    if (mask_out.has_value()) { TORCH_CHECK(mask_out->numel() == (int64_t)B * 70 && mask_out->scalar_type() == torch::kFloat32); mo = mask_out->data_ptr<float>(); }
    const unsigned long long* st = step.has_value() ? reinterpret_cast<const unsigned long long*>(step->data_ptr()) : nullptr;
    c10::cuda::CUDAGuard guard(params.device());
    const float* ax = nullptr;
    if (aux.has_value()) { TORCH_CHECK(aux->is_cuda() && aux->scalar_type() == torch::kFloat32 && aux->numel() >= 13000); ax = aux->data_ptr<float>(); }
    float* dp = nullptr;
    if (det_partials.has_value()) {
      const int ctas = cluster > 1 ? B * cluster : (max_ctas > 0 ? std::min(B, max_ctas) : B);   // CTAs of the step grid
      TORCH_CHECK(det_partials->is_cuda() && det_partials->scalar_type() == torch::kFloat32 &&
                  det_partials->numel() >= (int64_t)std::max(1, ctas) * 21888, "det_partials: [ctas, 21888] fp32");
      dp = det_partials->data_ptr<float>();
    }
    float* fp = nullptr;
    if (factors.has_value()) {
      // per-sample fc1 factors instead of fc1.weight in the slots (summed by reduce_sgd); one CTA per sample group only
      TORCH_CHECK(dp != nullptr && cluster <= 1, "factors need det_partials and cluster 1");
      TORCH_CHECK(factors->is_cuda() && factors->scalar_type() == torch::kFloat32 && factors->numel() >= (int64_t)std::max(1, B) * 384,
                  "factors: [B, 384] fp32");
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
  }, py::arg("params"), py::arg("grads"), py::arg("x"), py::arg("target"), py::arg("loss_acc"), py::arg("out_logp"),
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
                         c10::optional<torch::Tensor> grads, int64_t grad_stride, py::object lr_schedule) {
    // one-GPU optimizer step from convnet_step(..., det_partials=slots, factors=factors): the local gradient is summed from
    // the first n_slots slots and n_samples factor rows in a fixed order, then SGD is applied to it.  The gradient bucket is
    // not read; given `grads`, its other-parity half is re-zeroed like allreduce_sgd does, so a bucket step may follow.
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
    c10::cuda::CUDAGuard guard(params.device());
    ck_cuda(b2_reduce_sgd_launch(params.data_ptr<float>(), momentum.data_ptr<float>(), st, dc, (float)lr, (float)mu, ax, la, nullptr,
                                 slots.data_ptr<float>(), n_slots, factors.data_ptr<float>(), n_samples, g, grad_stride, &sched,
                                 cur_stream()),
            "reduce_sgd launch");
  }, py::arg("slots"), py::arg("n_slots"), py::arg("factors"), py::arg("n_samples"), py::arg("params"), py::arg("momentum"),
     py::arg("step"), py::arg("done_counter"), py::arg("lr"), py::arg("mu"), py::arg("aux") = py::none(), py::arg("loss_acc") = py::none(),
     py::arg("grads") = py::none(), py::arg("grad_stride") = 0, py::arg("lr_schedule") = py::none());
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
  m.def("gemm_bf16", [](torch::Tensor a, torch::Tensor b, c10::optional<torch::Tensor> bias, bool relu, bool out_bf16) {
    // C[M,N] = A[M,K] @ B[N,K]^T (+bias) (relu) ; A,B bf16 row-major (K contiguous)
    check_cuda_contig(a, "a"); check_cuda_contig(b, "b");
    TORCH_CHECK(a.scalar_type() == torch::kBFloat16 && b.scalar_type() == torch::kBFloat16, "bf16 operands");
    TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && a.size(1) == b.size(1), "A[M,K], B[N,K]");
    const int M = (int)a.size(0), K = (int)a.size(1), N = (int)b.size(0);
    TORCH_CHECK(K % 8 == 0, "K must be a multiple of 8 (16-byte rows for TMA)");
    const float* bp = nullptr;
    if (bias.has_value()) { TORCH_CHECK(bias->is_cuda() && bias->scalar_type() == torch::kFloat32 && bias->numel() == N); bp = bias->data_ptr<float>(); }
    auto c = torch::empty({M, N}, a.options().dtype(out_bf16 ? torch::kBFloat16 : torch::kFloat32));
    c10::cuda::CUDAGuard guard(a.device());
    int rc = b2_gemm_bf16_launch(a.data_ptr(), b.data_ptr(), c.data_ptr(), bp, M, N, K, relu, out_bf16, cur_stream());
    if (rc != 0) throw std::runtime_error(std::string("gemm_bf16: ") + b2_gemm_last_error());
    return c;
  }, py::arg("a"), py::arg("b"), py::arg("bias") = py::none(), py::arg("relu") = false, py::arg("out_bf16") = true);

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
                    c10::optional<torch::Tensor>, py::object>(),
           py::arg("loader"), py::arg("params"), py::arg("momentum"), py::arg("grads"), py::arg("grad_ptrs"),
           py::arg("sig_ptrs"), py::arg("step"), py::arg("done_counter"), py::arg("loss_acc"), py::arg("in_dev"),
           py::arg("raw_u8"), py::arg("training"), py::arg("rank"), py::arg("world"), py::arg("seed"),
           py::arg("sample_base"), py::arg("grad_stride"), py::arg("lr"), py::arg("mu"), py::arg("p_drop"),
           py::arg("max_in_flight") = 3, py::arg("cluster") = 1, py::arg("aux") = torch::Tensor(),
           py::arg("inbox") = std::vector<unsigned long long>(), py::arg("loss_hist") = torch::Tensor(),
           py::arg("wire_bf16") = false, py::arg("grad_slots") = py::none(),
           py::arg("factors") = py::none(), py::arg("lr_schedule") = py::none(), py::keep_alive<1, 2>())
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
