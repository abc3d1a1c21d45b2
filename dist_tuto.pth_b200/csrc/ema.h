// The exponential moving average of a model's weights (FlatEMA, ops/optim.py): one launch of ema_kernel (ema.cu) updates
// every entry of a device table built once, when the FlatEMA is constructed (the `ema_table` binding).
//
// An entry is one pair of fp32 arrays of n elements: an EMA array and the live values it follows -- a bucket's parameter flat,
// or when the optimizer is sharded this rank's slice [lo, hi) of the padded flat, or one fp32 buffer (BatchNorm statistics).
// Elements [0, head) and [head + 4 * n_vec, n) are done by scalar code, [head, head + 4 * n_vec) as 16-byte vectors, so
// `head` makes both arrays 16-byte aligned there.  An entry whose two arrays are not aligned alike is all scalar
// (head = n, n_vec = 0).  vec_begin / scalar_begin are the entry's first index in the concatenated vectors / scalars of all
// entries, ascending, so a thread finds its entry by a binary search.
//
// Per element (torch's lerp, ATen/native/Lerp.h, with torch's roundings and no flush of subnormals):
//   copy:  e = p
//   lerp:  w < 0.5:  e = fma(w, p - e, e);   otherwise  e = fma(-(p - e), 1 - w, p)   (1 - w in fp32)
// with w = fp32(1 - decay).  The build flushes fp32 subnormals (--use_fast_math), so these three operations are inline PTX
// without .ftz.
//
// No communication.  With a sharded optimizer the owned slice of the parameters was written by this rank's own exchange
// kernel, and the EMA reads that slice only, so no peer memory is read.  The kernel is ordered after the sharded exchanges
// and the unsharded updates because optimizer.step() (and DistributedDataParallel.finish()) run before FlatEMA.update() on
// the same stream.
#pragma once
#include <cstdint>

namespace b2 {

struct EmaEntry {
  float* ema;
  const float* live;
  long long n;              // elements
  long long head;           // scalar elements before the vectors
  long long n_vec;          // 16-byte vectors from element head
  long long vec_begin;      // first index of this entry's vectors among all entries' vectors
  long long scalar_begin;   // first index of this entry's n - 4 * n_vec scalars among all entries' scalars
  long long pad;
};
static_assert(sizeof(EmaEntry) == 64, "EmaEntry is 8 int64 words, as the ema_table binding writes it");

// ema_update's modes
enum EmaMode : int { EMA_LERP = 0, EMA_COPY = 1 };

}  // namespace b2
