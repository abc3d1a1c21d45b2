// The device state of a capturable FlatSGD / FlatAdamW (ops/optim.py, capturable=True), shared by the kernels and the host
// bindings: the hyper-parameter table the host uploads (FlatHyper) and the scalar block the update kernels read (FlatScalars),
// which flat_scalars_kernel (flat_scalars.cu) fills from the table and the device step counter.  The contract is in
// flat_scalars.cuh.
#pragma once
#include "adamw.h"
#include "lr_schedule.h"
#include "param_groups.h"

namespace b2 {

// What the host knows in fp64 and uploads with one stream-ordered copy: the schedule, the AdamW constants and every group's
// base lr and weight decay.  Without parameter groups there is one group, the optimizer's own lr / weight_decay.
struct FlatHyper {
  LrSchedule sched;            // kind LRS_NONE: the base lr as it is
  double beta1, beta2, eps;    // FlatAdamW (FlatSGD: 0)
  int n_groups;                // 1..kMaxGroups
  double lr[kMaxGroups];
  double wd[kMaxGroups];
};

// The scalars of ONE update, laid out as the by-value arguments of the existing instances take them, each rounded once to fp32:
//   lr, wd        sgd_flat / sgd_flat_clip / sharded_sgd (the last group's: the optimizer's own lr and weight decay)
//   adamw         adamw_flat / sharded_adamw, and the shared five of the grouped AdamW instances (decay and step_size of the
//                 last group)
//   sgd           the grouped SGD instances (every group's lr and wd)
//   adamw_groups  the grouped AdamW instances (every group's 1 - lr*wd and lr / (1 - beta1^t))
// Groups at and beyond n_groups are left as they are.
struct FlatScalars {
  float lr, wd;
  AdamwScalars adamw;
  SgdGroups sgd;
  AdamwGroups adamw_groups;
};

}  // namespace b2
