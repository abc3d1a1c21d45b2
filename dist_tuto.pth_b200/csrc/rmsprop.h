// The scalars of one RMSprop update (rmsprop_device.cuh), shared by the kernels and the host bindings.  The host computes
// them in fp64 from the hyper-parameters and rounds each once to fp32.
#pragma once

namespace b2 {

struct RmspropScalars {
  float lr;          // the update's lr (scheduled); grouped and capturable instances take it from the group / the block
  float wd;          // coupled weight decay: g + wd * p (same sources as lr)
  float alpha;       // the square average's smoothing constant
  float c;           // 1 - alpha: the weight of g * g and of the centered average's lerp
  float eps;
  float mu;          // momentum
  int centered;      // 1: the grad_avg state exists and the update is centered
  int momentum;      // 1: the momentum_buffer state exists (mu > 0)
};

}  // namespace b2
