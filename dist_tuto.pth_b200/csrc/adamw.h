// The scalars of one AdamW update (adamw_device.cuh), shared by the kernels and the host bindings.  The host computes them
// in fp64 from the hyper-parameters and the update index t and rounds each once to fp32.
#pragma once

namespace b2 {

struct AdamwScalars {
  float decay;       // 1 - lr * weight_decay
  float w1;          // 1 - beta1 (the lerp weight)
  float beta2, c2;   // beta2, 1 - beta2
  float step_size;   // lr / (1 - beta1^t)
  float sbc2;        // sqrt(1 - beta2^t)
  float eps;
};

}  // namespace b2
