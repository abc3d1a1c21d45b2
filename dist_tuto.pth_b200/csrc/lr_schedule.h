// Learning-rate schedule of the optimizer kernels: the device (and host C++) twin of ops/optim.LRSchedule.
//
// The lr of an update is a closed-form function of the device step counter's value when the update runs (the number of
// updates applied before it), so captured graphs and the native executor's launches replay the same arguments and still
// follow the schedule.  Every operation is an explicitly rounded fp64 one (no fused multiply-add on
// the device), and the product with the base lr is rounded to fp32 once: the device and LRSchedule.lr_at agree bit for
// bit except for the cosine, which the device takes as cospi(d / span) and the host as cos(pi * d / span); the two may
// differ in the last fp64 bits, and so the fp32 lr by at most one ulp.
//
// Plain C++ too: executor.cpp and bindings.cpp include this header, the kernels include it through sgd_device.cuh.
#pragma once

#ifdef __CUDACC__
#define B2_LRS_FN __host__ __device__ inline
#else
#define B2_LRS_FN inline
#endif

#include <math.h>

namespace b2 {

enum : int { LRS_NONE = 0, LRS_CONSTANT = 1, LRS_MULTISTEP = 2, LRS_COSINE = 3 };
constexpr int LRS_MAX_MILESTONES = 8;

// Zero-initialised (kind == LRS_NONE): no schedule, the kernels use the fp32 lr they were given as it is.
struct LrSchedule {
  int kind;                              // LRS_*
  int n_milestones;                      // LRS_MULTISTEP: milestones[0, n) are used
  long long warmup;                      // W: updates 0 .. W-1 ramp linearly from start to 1
  long long total;                       // LRS_COSINE: T > W, the factor stays at min_factor from update T on
  double start, gamma, min_factor;
  long long milestones[LRS_MAX_MILESTONES];   // LRS_MULTISTEP: absolute update indices, sorted
};

#if defined(__CUDA_ARCH__)
B2_LRS_FN double lrs_add(double a, double b) { return __dadd_rn(a, b); }
B2_LRS_FN double lrs_mul(double a, double b) { return __dmul_rn(a, b); }
B2_LRS_FN double lrs_div(double a, double b) { return __ddiv_rn(a, b); }
B2_LRS_FN float lrs_to_f32(double a) { return __double2float_rn(a); }
#else
B2_LRS_FN double lrs_add(double a, double b) { return a + b; }
B2_LRS_FN double lrs_mul(double a, double b) { return a * b; }
B2_LRS_FN double lrs_div(double a, double b) { return a / b; }
B2_LRS_FN float lrs_to_f32(double a) { return (float)a; }
#endif

// Multiplier of the base lr for the update that runs when the step counter reads `step`.
B2_LRS_FN double lr_schedule_factor(const LrSchedule& s, unsigned long long step) {
  const double k = (double)step;
  if ((long long)step < s.warmup)                            // f0 + (1 - f0) * s / W
    return lrs_add(s.start, lrs_div(lrs_mul(lrs_add(1.0, -s.start), k), (double)s.warmup));
  double f = 1.0;
  if (s.kind == LRS_MULTISTEP) {                             // gamma ** #{m <= s}, one multiplication per milestone passed
#ifdef __CUDA_ARCH__
#pragma unroll                                               // constant indices: the milestones stay in parameter space
#endif
    for (int i = 0; i < LRS_MAX_MILESTONES; ++i)
      if (i < s.n_milestones && s.milestones[i] <= (long long)step) f = lrs_mul(f, s.gamma);
  } else if (s.kind == LRS_COSINE) {                         // min + (1 - min) * (1 + cos(pi * d / (T - W))) / 2
    const long long span = s.total - s.warmup;
    const long long d = (long long)step - s.warmup < span ? (long long)step - s.warmup : span;
#ifdef __CUDA_ARCH__
    const double c = cospi(lrs_div((double)d, (double)span));   // the argument is in [0, 1]: no large-argument reduction
#else
    const double c = cos(lrs_div(lrs_mul(3.141592653589793, (double)d), (double)span));
#endif
    f = lrs_add(s.min_factor, lrs_div(lrs_mul(lrs_add(1.0, -s.min_factor), lrs_add(1.0, c)), 2.0));
  }
  return f;
}

// fp32 lr of that update: base * factor rounded once (base itself when there is no schedule).
B2_LRS_FN float lr_schedule_lr(const LrSchedule& s, float base, unsigned long long step) {
  if (s.kind == LRS_NONE) return base;
  return lrs_to_f32(lrs_mul((double)base, lr_schedule_factor(s, step)));
}

}  // namespace b2
