// The argument block of the SyncBatchNorm kernels (csrc/batchnorm.cu), filled by the bindings.
#pragma once

namespace b2 {
namespace bn {

struct Args {
  const void* x;
  void* y;                // forward output
  const void* dy;
  void* dx;               // input gradient
  const void* w;          // weight (null: affine=False)
  const void* b;
  void* rmean;            // running stats (null: not tracked)
  void* rvar;
  void* gw;               // local grad_weight / grad_bias (null: not wanted)
  void* gb;
  int pw, pr;             // dtype codes of weight / bias / grads and of the running stats: 0 fp32, 1 bf16, 2 fp16
  const long long* nbt;   // num_batches_tracked when momentum is None (factor 1 / nbt), else null
  double momentum, eps;
  double* ex;             // exchange buffer, n_ex doubles
  int n_ex;
  double* part;           // [splits][2][C] CTA partials
  unsigned int* tickets;  // [tiles], zero between calls
  double* stats;          // [mean C | invstd C | global count]
  long long count;        // local elements per channel
  // geometry
  long long rows;         // channels-last: rows M; channel-first: vectors per channel (N x L/V)
  long long per_split;    // rows / vectors per split
  long long Lv;           // channel-first: vectors per (n, c) row
  int C, cv, cx, tiles;
};

}  // namespace bn
}  // namespace b2
