#!/bin/bash
# Race / memory checking of the hand-written kernels with compute-sanitizer (needs a GPU and the CUDA toolkit's
# compute-sanitizer; slow -- small shapes only).  Reports go to ${SANITIZE_OUT:-$TMPDIR/sanitize}.
#   memcheck : out-of-bounds / misaligned accesses
#   racecheck: shared-memory hazards (phase barriers of the fused ConvNet kernels, staging tiles of the tensor-core kernels)
#   synccheck: divergent / mismatched barriers (incl. named barriers and mbarrier use in the wgmma kernels)
# Coverage: per-sample kernel (1 CTA and 4-CTA cluster per sample), deterministic flush + det_reduce, the batched tensor-core
# engine (B = 2 eval: every kernel of the pipeline), sgd_flat, the TMA + wgmma GEMM (both kernels), reduce_sgd's instances (memcheck,
# the clip instance at a 3-CTA grid) and det_reduce; with 2 GPUs, memcheck of
# the push exchange and the all-reduce variants under `--target-processes all`.
set -u
cd "$(dirname "$0")/.."
OUT=${SANITIZE_OUT:-${TMPDIR:-/tmp}/sanitize}
mkdir -p "$OUT"
SEL1='test_convnet_loss_and_grads_match_autograd[16] or test_convnet_training_dropout or test_sgd_flat or test_tcgen05_gemm_matches_torch[128-64-64] or test_tcgen05_gemm_matches_torch[2500-2048-2056] or test_fused_trainer_uses_clusters_for_small_batches or test_deterministic_mode_is_bit_reproducible[32]'
for tool in memcheck racecheck synccheck; do
  timeout 1200 compute-sanitizer --tool $tool --error-exitcode 1 python -m pytest tests/test_gpu_kernels.py -q -m gpu -p no:cacheprovider -k "$SEL1" > "$OUT/${tool}_persample.txt" 2>&1
  echo "$tool per-sample rc=$?" | tee -a "$OUT/summary.txt"; grep -E "ERROR SUMMARY|passed|failed" "$OUT/${tool}_persample.txt" | tail -3 | tee -a "$OUT/summary.txt"
  timeout 1200 compute-sanitizer --tool $tool --error-exitcode 1 python -m pytest tests/test_gpu_batched.py -q -m gpu -p no:cacheprovider -k "test_every_stage_matches_the_rounding_exact_model[2-False] or test_uint8" > "$OUT/${tool}_batched.txt" 2>&1
  echo "$tool batched rc=$?" | tee -a "$OUT/summary.txt"; grep -E "ERROR SUMMARY|passed|failed" "$OUT/${tool}_batched.txt" | tail -3 | tee -a "$OUT/summary.txt"
done
SEL2='test_every_grid_reduces_in_the_model_order[5x24] or test_every_instance_matches_the_model_with_guard_bands[wd+nesterov+cosine] or test_every_instance_matches_the_model_with_guard_bands[clip+wd+nesterov] or test_det_reduce_sums_in_slot_order[33]'
timeout 1200 compute-sanitizer --tool memcheck --error-exitcode 1 python -m pytest tests/test_gpu_reduce_sgd_order.py -q -m gpu -p no:cacheprovider -k "$SEL2" > "$OUT/memcheck_reduce_sgd.txt" 2>&1
echo "memcheck reduce_sgd rc=$?" | tee -a "$OUT/summary.txt"; grep -E "ERROR SUMMARY|passed|failed" "$OUT/memcheck_reduce_sgd.txt" | tail -3 | tee -a "$OUT/summary.txt"
if [ "$(nvidia-smi -L | wc -l)" -ge 2 ]; then
  B200DIST_STRESS_ITERS=200 timeout 1500 compute-sanitizer --tool memcheck --target-processes all --error-exitcode 1 python -m pytest tests/test_gpu_multi.py -q -p no:cacheprovider -k "test_push_exchange_equals_barrier_exchange or test_symmetric_allreduce_all_variants_vs_nccl" > "$OUT/memcheck_multigpu.txt" 2>&1
  echo "memcheck multi-GPU rc=$?" | tee -a "$OUT/summary.txt"; grep -E "ERROR SUMMARY|passed|failed" "$OUT/memcheck_multigpu.txt" | tail -4 | tee -a "$OUT/summary.txt"
fi
