// Parameter groups of FlatSGD / FlatAdamW (ops/optim.py) on the device, shared by the kernels and the host bindings: the
// per-group scalars, passed by value in the kernel arguments (no copy to the device, no host synchronisation), for at most
// kMaxGroups groups.  The kernels find a vector's group in a group map with one uint8 id per 16-byte fp32 parameter vector:
// GradBucket lays every tensor out at a multiple of 4 elements, so a parameter vector never straddles two tensors.  The host
// builds the map once at construction and checks every id against the number of groups there.
#pragma once

namespace b2 {

constexpr int kMaxGroups = 64;

// FlatSGD: lr and weight decay of each group, rounded once to fp32 by the host
struct SgdGroups {
  float lr[kMaxGroups];
  float wd[kMaxGroups];
};

// FlatAdamW: the two AdamwScalars that depend on lr or weight decay, per group (1 - lr*wd and lr / (1 - beta1^t), computed in
// fp64 and rounded once); the other five stay shared
struct AdamwGroups {
  float decay[kMaxGroups];
  float step_size[kMaxGroups];
};

}  // namespace b2
