// The step counter and scalar block of a capturable FlatSGD / FlatAdamW (flat_scalars.cuh): one CTA per call, one thread per
// parameter group.
#include "flat_scalars.cuh"

namespace b2 {

// advance = 1: counter += 1, then the block of the update run at the new count; advance = 0: the block of the update run at
// the current count.  The only writer of the counter and the block while it runs.  kGated: the advance after a step
// GradScaler may have skipped; with *found_inf != 0 the counter and the block stay as they are, so the skipped step counts
// for neither the schedule nor the bias corrections.
template <bool kGated>
__global__ void __launch_bounds__(kMaxGroups) flat_scalars_kernel(const FlatHyper* __restrict__ h, unsigned long long* counter,
                                                                  FlatScalars* __restrict__ out, int advance,
                                                                  const float* found_inf) {
  if constexpr (kGated) {
    if (__ldg(found_inf) != 0.f) return;
  }
  __shared__ unsigned long long s_step;
  if (threadIdx.x == 0) s_step = *counter + (unsigned long long)advance;
  __syncthreads();
  const unsigned long long s = s_step;
  if (threadIdx.x == 0 && advance) *counter = s;
  const int g = threadIdx.x;
  const int n = h->n_groups;
  if (g >= n) return;
  const double b1 = h->beta1, b2 = h->beta2, wd = h->wd[g];
  const float lr = lr_schedule_lr(h->sched, __double2float_rn(h->lr[g]), s);
  const double p1 = flat_pow(b1, s + 1ull), p2 = flat_pow(b2, s + 1ull);
  const float decay = __double2float_rn(__dadd_rn(1.0, -__dmul_rn((double)lr, wd)));
  const float step_size = __double2float_rn(__ddiv_rn((double)lr, __dadd_rn(1.0, -p1)));
  out->sgd.lr[g] = lr;
  out->sgd.wd[g] = __double2float_rn(wd);
  out->adamw_groups.decay[g] = decay;
  out->adamw_groups.step_size[g] = step_size;
  if (g == n - 1) {
    out->lr = lr;
    out->wd = __double2float_rn(wd);
    AdamwScalars a;
    a.decay = decay;
    a.w1 = __double2float_rn(__dadd_rn(1.0, -b1));
    a.beta2 = __double2float_rn(b2);
    a.c2 = __double2float_rn(__dadd_rn(1.0, -b2));
    a.step_size = step_size;
    a.sbc2 = __double2float_rn(__dsqrt_rn(__dadd_rn(1.0, -p2)));
    a.eps = __double2float_rn(h->eps);
    out->adamw = a;
  }
}

}  // namespace b2

extern "C" {

// found_inf (fp32 on the device, or null): the gated advance; it needs advance != 0.
int b2_flat_scalars_launch(const b2::FlatHyper* table, unsigned long long* counter, b2::FlatScalars* block, int advance,
                           const float* found_inf, cudaStream_t stream) {
  if (table == nullptr || counter == nullptr || block == nullptr) return (int)cudaErrorInvalidValue;
  if (found_inf != nullptr && !advance) return (int)cudaErrorInvalidValue;
  if (found_inf != nullptr)
    b2::flat_scalars_kernel<true><<<1, b2::kMaxGroups, 0, stream>>>(table, counter, block, 1, found_inf);
  else
    b2::flat_scalars_kernel<false><<<1, b2::kMaxGroups, 0, stream>>>(table, counter, block, advance ? 1 : 0, nullptr);
  return (int)cudaGetLastError();
}

}  // extern "C"
