// Shared between the fused ConvNet kernels (convnet.cu: one CTA per sample; convnet_cluster.cu: one cluster per sample).
#pragma once
#include <cuda_runtime.h>

#include "sgd_device.cuh"

namespace cn {

constexpr int W1 = 0, B1 = 252, W2 = 264, B2 = 5264, W3 = 5284, B3 = 21284, W4 = 21336, B4 = 21836;
constexpr int NPAR = 21848;

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

struct Args {
  const float* params;      // flat fp32 [NPAR]
  float* grads;             // flat fp32 [NPAR], accumulated with red.add (caller keeps it zeroed)
  const void* x;            // [B,1,28,28] fp32 (normalised) or uint8 (raw, normalised here)
  const long long* target;  // [B]
  float* loss_acc;          // [0] += sum_b nll_b * inv_bsz ; [1] += #correct   (may be null)
  float* out_logp;          // [B,10] log-probabilities (may be null)
  float* mask_out;          // [B,70] dropout scales actually applied (debug/tests; may be null)
  const unsigned long long* step;   // device step counter (RNG offset); may be null -> 0
  unsigned long long seed;
  long long sample_base;    // global index of sample 0 (rank * bsz): decorrelates ranks
  int B;
  int x_u8;
  int training;             // dropout on/off
  int backward;             // compute gradients
  float inv_bsz;            // 1 / local batch (nll_loss mean)
  float p_drop;
  float mean, inv_std;      // uint8 normalisation
  long long grad_stride;    // elements between the two gradient buckets (0: single bucket); bucket = step & 1
  const float* aux;         // optional: conv2.weight pre-arranged by the SGD kernel as [w2f 5000 | w2b 8000] (see sgd.cu)
  float* det_partials;      // per-CTA slots: CTA i stores its gradient sums and loss terms to det_partials + i * DET_STRIDE
                            // (plain stores) instead of red.add-ing into the bucket; they are summed in slot order afterwards,
                            // by det_reduce_kernel or, with `factors`, by the reduction of convnet_reduce.cuh
  float* factors;           // with det_partials: sample b stores its fc1 factors dh (50) and p2 (320) to factors + b * FAC_STRIDE
                            // instead of dh (x) p2 into its slot; the slot's fc1.weight range is then left unwritten
  unsigned long long* phase_ts;   // optional phase timestamps (sgd_device.cuh: TS_STEPS); nullptr: off
  int input_ready;          // x and target are not written by the kernel this one waits on (griddepcontrol.wait): the kernel
                            // may read them before that wait returns
};

constexpr int DET_STRIDE = 21888;   // = NPAR_ALLOC of ops/convnet_fused.py
constexpr int FAC_STRIDE = 384, FAC_P2 = 64;   // per-sample fc1 factors: dh at [0, 50), p2 at [FAC_P2, FAC_P2 + 320)

constexpr int AUX_W2F = 0, AUX_W2B = 5000, AUX_TOTAL = 13000;

// relu(pool(conv1)) lives in shared memory as [10 planes][12 rows][12 cols] with row stride 13 and plane stride 161: with these
// strides the 32 (input channel, kernel row) work items of a warp in the conv2 weight-gradient phase hit 32 distinct banks
// (dense 12/144 strides gave 4.8-way conflicts there -- 41 % of all excess shared-memory wavefronts of the kernel).
constexpr int P1_ROW = 13, P1_PLANE = 161, P1_SIZE = (10 * P1_PLANE + 3) / 4 * 4;   // keeps the next shared array 16-byte aligned
// The zero-padded conv2-output gradient [20][16][16] uses row stride 20 / plane stride 324 and is read as float2 pairs:
// 9720 -> 3240 shared-memory wavefronts per sample in the conv2 data-gradient phase (dense 16/256 strides, scalar loads).
constexpr int DC_ROW = 20, DC_PLANE = 324, DC_SIZE = 20 * DC_PLANE;
__host__ __device__ constexpr int p1_idx(int c, int y, int x) { return c * P1_PLANE + y * P1_ROW + x; }
__host__ __device__ constexpr int p1_of(int o) { return (o / 144) * P1_PLANE + ((o % 144) / 12) * P1_ROW + (o % 12); }   // o = c*144 + y*12 + x

}  // namespace cn
