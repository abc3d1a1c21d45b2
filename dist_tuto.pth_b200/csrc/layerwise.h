// FlatLAMB / FlatLARS (ops/optim.py): the chunk table of a flat bucket and the arguments of the layer-wise kernels
// (layerwise.cu), shared by the kernels and the host bindings.
#pragma once
#include <cstddef>

namespace b2 {

// Every tensor's segment [offset, offset + numel) of a bucket is cut into chunks of at most kLwChunk elements; no chunk
// crosses a tensor boundary.  One CTA of kLwThreads threads takes one chunk at a time (16 float4 vectors per thread).
constexpr int kLwThreads = 256;
constexpr long long kLwChunk = 16384;
// The table, one int64 array: n_chunks rows (start, length, tensor), then n_tensors rows (first chunk, chunks, adapt).
// A tensor without elements has no chunk; its ratio is never written.
constexpr int kLwRow = 3;

struct LwArgs {
  float* p;                 // parameters
  float* g;                 // averaged gradients
  float* m;                 // LAMB: exp_avg; LARS: momentum
  float* v;                 // LAMB: exp_avg_sq; LARS: unused
  size_t n;                 // elements of the flats
  const long long* table;   // n_chunks * kLwRow + n_tensors * kLwRow
  int n_chunks, n_tensors;
  float* partials;          // [2 * n_chunks]: (sum of p^2, sum of u^2 or g^2) per chunk
  unsigned int* tickets;    // [n_tensors], zero between calls (the last CTA of a tensor re-zeroes its ticket)
  double* sums;             // [2 * n_tensors]: the tensor's two sums of squares, fp64
  float* ratios;            // [n_tensors]: the trust ratio of the last update
  int zero_grad;
  // LAMB (update t): w1 = 1 - beta1, beta2, c2 = 1 - beta2, sbc2 = sqrt(1 - beta2^t), eps, rbc1 = 1 / (1 - beta1^t), lr, wd
  // LARS: lr, mu (momentum), wd, nesterov; eta (trust coefficient), eps and wd again in fp64 for the ratio
  float w1, beta2, c2, sbc2, eps, rbc1, lr, wd, mu;
  int nesterov;
  double eta64, wd64, eps64;
  // clipping: g *= clip_coef(sqrt(sum of sqnorms[0, n_buckets))), as adamw_flat_kernel<true> does
  const double* sqnorms;
  int n_buckets;
  float max_norm;
  float* grad_norm_out;
  // fp16 loss scaling: GradScaler's scale S on the device (fp32), or null; the scaled instances read g * fp32(1 / double(S))
  const float* grad_scale;
};

}  // namespace b2
