// The momentum SGD step of four elements, shared by sgd_flat_grouped_kernel (sgd.cu) and the sharded kernel's SGD instances
// (sharded_sgd.cu), and the group scalars of param_groups.h.
#pragma once
#include <cstdint>
#include "param_groups.h"

namespace b2 {

// momentum SGD on four elements, the fmaf sequence of sgd_flat_kernel (sgd.cu)
template <bool kNesterov>
__device__ __forceinline__ void sgd4(float4& p, float4& m, float4 g, float lr, float mu, float wd) {
  g.x = fmaf(wd, p.x, g.x); g.y = fmaf(wd, p.y, g.y); g.z = fmaf(wd, p.z, g.z); g.w = fmaf(wd, p.w, g.w);
  m.x = fmaf(mu, m.x, g.x); m.y = fmaf(mu, m.y, g.y); m.z = fmaf(mu, m.z, g.z); m.w = fmaf(mu, m.w, g.w);
  float4 d = m;
  if (kNesterov) {
    d.x = fmaf(mu, m.x, g.x); d.y = fmaf(mu, m.y, g.y); d.z = fmaf(mu, m.z, g.z); d.w = fmaf(mu, m.w, g.w);
  }
  p.x = fmaf(-lr, d.x, p.x); p.y = fmaf(-lr, d.y, p.y); p.z = fmaf(-lr, d.z, p.z); p.w = fmaf(-lr, d.w, p.w);
}

}  // namespace b2
