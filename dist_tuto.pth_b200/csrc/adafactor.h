// FlatAdafactor (ops/optim.py): the chunk table of a flat bucket and the arguments of the Adafactor kernels (adafactor.cu),
// shared by the kernels and the host bindings.
#pragma once
#include <cstddef>

#include "param_groups.h"

namespace b2 {

// A tensor of dim > 1 is factored over its last two dimensions: B slices (the product of the leading dimensions) of R rows
// and C columns.  Element (b, r, c) lives at  offset + lead(b) + r * sR + c * sC  of the flat, with lead(b) from the
// leading sizes and strides (row-major over the leading dimensions), so any dense layout works, channels_last included.
// A tensor of dim <= 1 is one slice of one row of numel contiguous columns.
//
// The table cuts every tensor into chunks of at most kAfChunk elements, none crossing a tensor boundary.  A chunk is a box
// [b0, b0 + nb) x [r0, r0 + nr) x [c0, c0 + nc) of the tensor's logical index space:
//   * unfactored: nb = nr = 1 and a run of columns;
//   * factored with R * C <= kAfChunk ("whole"): floor(kAfChunk / (R * C)) whole slices, so the chunk owns complete rows,
//     columns and slices and finishes their statistics itself;
//   * factored otherwise ("tiled"): one tile of TR x TC of one slice, chunks in (b, tile row, tile column) order; the row
//     and column sums of g^2 go out as per-tile partials that the tensor's last CTA adds up.
constexpr int kAfThreads = 256;
constexpr long long kAfChunk = 8192;
constexpr long long kAfTileCols = 256;      // a tile's width before it is widened to fill the chunk
// Shared memory of the stats kernel: a chunk's gradients, rows padded to an odd pitch (nc | 1), at most kAfChunk * 3 / 2
// floats (nc = 2 gives pitch 3).
constexpr int kAfSmemFloats = (int)(kAfChunk * 3 / 2);
constexpr int kAfMaxLead = 4;               // leading dimensions after merging the ones that merge
// Chunk rows: (tensor, b0, nb, r0, nr, c0, nc, 0).
constexpr int kAfChunkRow = 8;
// Tensor rows, kAfTensorRow int64 each:
enum : int {
  AF_OFFSET = 0,      // first element of the tensor's segment of the flat
  AF_STATE,           // first element of its state: row_var [B*R] then col_var [B*C], or variance [numel]
  AF_B, AF_R, AF_C,   // slices, rows, columns (unfactored: 1, 1, numel)
  AF_SR, AF_SC,       // row and column strides (unfactored: 0, 1)
  AF_FIRST, AF_COUNT, // its chunks: [first, first + count)
  AF_FACTORED,        // 1: dim > 1
  AF_GROUP,           // parameter group (lr, weight decay) in [0, n_groups)
  AF_WHOLE,           // factored: 1 when its chunks hold whole slices
  AF_TR, AF_TC,       // tiled: the tile's rows and columns
  AF_RC,              // tiled: first row partial; B*R*ceil(C/TC) row partials, then B*C*ceil(R/TR) column partials
  AF_MEAN,            // factored: first of its B clamped row_var means
  AF_NLEAD,           // leading dimensions after merging, 0..kAfMaxLead
  AF_LSIZE,           // kAfMaxLead sizes
  AF_LSTRIDE = AF_LSIZE + kAfMaxLead,   // kAfMaxLead strides
  kAfTensorRow = AF_LSTRIDE + kAfMaxLead
};

struct AfArgs {
  float* p;                 // parameters
  float* g;                 // averaged gradients
  float* state;             // row_var / col_var / variance of every tensor (AF_STATE)
  size_t n;                 // elements of the parameter and gradient flats
  const long long* table;   // n_chunks * kAfChunkRow + n_tensors * kAfTensorRow
  int n_chunks, n_tensors;
  float* partials;          // [2 * n_chunks]: sum of p^2, then sum of u^2, per chunk
  float* rc;                // the tiled tensors' row and column partials of g^2
  float* means;             // the factored tensors' clamped row_var means, one per slice
  unsigned int* tickets;    // [n_tensors], zero between calls (the last CTA of a tensor re-zeroes its ticket)
  double* alpha;            // [n_tensors]: max(eps2, ||p|| / sqrt(numel)) * rho_t of this update
  float* step;              // [n_tensors]: fp32(-alpha / max(1, ||u|| / (sqrt(numel) * d))) of this update
  int zero_grad;
  // update t: w = fp32(t ** beta2_decay) (the lerp weight), eps1 and fp32(eps1 * eps1), eps2, d
  float w, eps1, eps1sq;
  double eps2, d;
  // per group: rho_t = min(lr, 1 / sqrt(t)) in fp64 and the decay fp32(1 - lr * weight_decay), lr the scheduled lr
  int n_groups;
  double rho[kMaxGroups];
  float decay[kMaxGroups];
  // clipping: g *= clip_coef(sqrt(sum of sqnorms[0, n_buckets))), as the layer-wise kernels do
  const double* sqnorms;
  int n_buckets;
  float max_norm;
  float* grad_norm_out;
  // fp16 loss scaling: GradScaler's scale S on the device (fp32), or null; the scaled instances read g * fp32(1 / double(S))
  const float* grad_scale;
};

}  // namespace b2
