// The grid of the sharded step launchers (sharded_sgd.cu, sharded_layerwise.cu).  The per-block barriers pair block b of
// every rank, so the grid is a function of the bucket, the world and max_blocks only: the same on every rank.
#pragma once
#include <cstddef>
#include <cuda_runtime.h>
#include "common.cuh"

// The two-shot all-reduce's grid: ceil(ceil(slice / 512) / 2) CTAs, at most max_blocks (B2_MAX_BLOCKS for max_blocks <= 0).
inline dim3 shard_grid(size_t n_vec, int world, int max_blocks) {
  constexpr size_t kThreads = 512;
  if (max_blocks <= 0 || max_blocks > B2_MAX_BLOCKS) max_blocks = B2_MAX_BLOCKS;
  size_t blocks = (n_vec / world + kThreads - 1) / kThreads;
  blocks = (blocks + 1) / 2;
  if (blocks < 1) blocks = 1;
  if (blocks > (size_t)max_blocks) blocks = (size_t)max_blocks;
  return dim3((unsigned)blocks);
}
