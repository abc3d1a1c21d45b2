// Local gradient of the per-sample step kernel (convnet.cu) from what its CTAs left in global memory with plain stores:
//   * one slot per CTA (det_partials layout): that CTA's sums of every parameter gradient except fc1.weight, and its loss terms;
//   * per-sample fc1 factors dh_b (50) and p2_b (320): fc1.weight's gradient is sum_b dh_b (x) p2_b, a 50 x 320 x B fp32 GEMM.
// Every sum runs in an order that depends only on the batch and the step grid (no atomics), so two runs are bit-equal.
#pragma once
#include "convnet_args.cuh"

namespace cn {

constexpr int RED_T = 512;
// Work units, dealt round robin to the CTAs of the reduction (unit u -> CTA u % n_cta):
//   units [0, RED_FC1_TILES): fc1.weight tiles of RJ output rows x RI inputs (RJ * RI / 4 vectors); a tile reads only its
//     dh and p2 columns (RKC samples per pass through shared memory) and splits the samples over RKS thread groups;
//   the rest: chunks of RV consecutive vectors of the other parameters; the slots are split over RSS thread groups, so a
//     thread has only a few independent loads in flight instead of one chain over all slots.
// Partial sums are combined in shared memory in group order.
// Load schedule: the inputs of a unit are read from L2, where the step kernel has just stored them, so what a unit costs is
// the number of dependent L2 round trips.  Every thread issues all of its loads of a unit (the caller's pre() loads, and per
// fc1 pass all its dh / p2 loads, per RSLOT_BATCH slots all its slot loads) before it uses any of them: one round trip per
// unit up to RKC samples and RSLOT_BATCH * RSS step CTAs.  The fc1 loads go to the RED_LOADERS threads of the sample groups,
// so the last warp is free for the loss sum of CTA 0.
constexpr int RJ = 10, RI = 32, RV = 20, RKC = 128;
constexpr int RED_TILE_VEC = RJ * RI / 4;                                  // 80 vectors per fc1 tile
constexpr int RED_FC1_TILES = (50 / RJ) * (320 / RI);                      // 50
constexpr int RED_OTHER = (NPAR - 16000) / 4;                              // 1462 vectors outside fc1.weight
constexpr int RED_UNITS = RED_FC1_TILES + (RED_OTHER + RV - 1) / RV;       // 124
constexpr int RKS = RED_T / RED_TILE_VEC, RSS = RED_T / RV;                // 6 sample groups, 25 slot groups
constexpr int RED_PART = RKS * RED_TILE_VEC > RSS * RV ? RKS * RED_TILE_VEC : RSS * RV;
constexpr int RED_LOADERS = RKS * RED_TILE_VEC;                            // 480 threads load an fc1 pass
constexpr int RDH_PER_T = (RKC * (RJ / 2) + RED_LOADERS - 1) / RED_LOADERS;  // 2 float2 of dh per loader and pass
constexpr int RP2_PER_T = (RKC * (RI / 4) + RED_LOADERS - 1) / RED_LOADERS;  // 3 float4 of p2
constexpr int RSLOT_BATCH = (RKC + RSS - 1) / RSS;                         // 6 slots per thread and batch of loads
static_assert(RED_LOADERS <= RED_T - 32, "the last warp loads no fc1 factors");
static_assert(50 % RJ == 0 && 320 % RI == 0 && RJ % 2 == 0 && RI % 4 == 0, "fc1 tiles must cover fc1.weight in vectors");
static_assert(W3 % 4 == 0 && FAC_STRIDE % 4 == 0 && FAC_P2 % 4 == 0 && FAC_P2 >= 50 && FAC_P2 + 320 <= FAC_STRIDE, "factor layout");

struct RedSmem {
  float dh[RKC][RJ];
  float4 p2[RKC][RI / 4];
  float4 part[RED_PART];
};

__device__ __forceinline__ void f4_add(float4& a, const float4 b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }

// CTA `cta` of `n_cta` produces the final local gradient of its units: for every float4 vector v of the flat gradient that the
// CTA owns, one thread calls h = pre(v) before the unit's loads (so whatever the caller needs besides the gradient is in
// flight with them) and emit(v, g, h) at the end, with g in registers.  n_slots = CTAs of the step grid, n_samples = batch.
// Thread 0 calls at(point, u) during unit u: RED_AT_ISSUED once its loads of the unit are in flight and before it waits on
// any (work that needs a load of its own, and must be done before the unit's first barrier, goes there),
// RED_AT_LOADED right after the unit's first barrier (its global loads have landed), RED_AT_EMITTED after its emit.
// Contains barriers: every thread of the CTA calls it.
enum : int { RED_AT_ISSUED = 0, RED_AT_LOADED, RED_AT_EMITTED };
template <class Pre, class Emit, class At>
__device__ __forceinline__ void reduce_local_grad(const float* __restrict__ slots, int n_slots, const float* __restrict__ fac,
                                                  int n_samples, int cta, int n_cta, RedSmem& s, Pre&& pre, Emit&& emit,
                                                  At&& at) {
  const int tid = threadIdx.x;
  for (int u = cta; u < RED_UNITS; u += n_cta) {
    if (u != cta) __syncthreads();                     // shared memory of the previous unit is consumed
    decltype(pre(0)) held{};
    if (u < RED_FC1_TILES) {
      const int j0 = (u / (320 / RI)) * RJ, i0 = (u % (320 / RI)) * RI;
      const int vec = tid % RED_TILE_VEC, ks = tid / RED_TILE_VEC;
      const int jj = vec / (RI / 4), ii4 = vec % (RI / 4);
      const int v = W3 / 4 + (j0 + jj) * 80 + i0 / 4 + ii4;
      if (tid < RED_TILE_VEC) held = pre(v);
      float4 total = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int k0 = 0;; k0 += RKC) {                  // one pass at least, so at() sees every point of the unit
        const int kn = min(RKC, n_samples - k0);
        if (k0 > 0) __syncthreads();                   // the previous pass is consumed
        const float* f0 = fac + (size_t)k0 * FAC_STRIDE;
        // element e of the pass: sample e / (columns), column e % (columns); loader tid takes e = tid + i * RED_LOADERS
        float2 d[RDH_PER_T];
        float4 p[RP2_PER_T];
#pragma unroll
        for (int i = 0; i < RDH_PER_T; ++i) {
          const int e = tid + i * RED_LOADERS, k = e / (RJ / 2), q = e - k * (RJ / 2);
          if (tid < RED_LOADERS && e < kn * (RJ / 2))
            d[i] = __ldcg(reinterpret_cast<const float2*>(f0 + (size_t)k * FAC_STRIDE + j0) + q);
        }
#pragma unroll
        for (int i = 0; i < RP2_PER_T; ++i) {
          const int e = tid + i * RED_LOADERS, k = e / (RI / 4), q = e - k * (RI / 4);
          if (tid < RED_LOADERS && e < kn * (RI / 4))
            p[i] = __ldcg(reinterpret_cast<const float4*>(f0 + (size_t)k * FAC_STRIDE + FAC_P2 + i0) + q);
        }
        if (k0 == 0 && tid == 0) at(RED_AT_ISSUED, u);
#pragma unroll
        for (int i = 0; i < RDH_PER_T; ++i) {
          const int e = tid + i * RED_LOADERS, k = e / (RJ / 2), q = e - k * (RJ / 2);
          if (tid < RED_LOADERS && e < kn * (RJ / 2)) { s.dh[k][2 * q] = d[i].x; s.dh[k][2 * q + 1] = d[i].y; }
        }
#pragma unroll
        for (int i = 0; i < RP2_PER_T; ++i) {
          const int e = tid + i * RED_LOADERS, k = e / (RI / 4), q = e - k * (RI / 4);
          if (tid < RED_LOADERS && e < kn * (RI / 4)) s.p2[k][q] = p[i];
        }
        __syncthreads();
        if (k0 == 0 && tid == 0) at(RED_AT_LOADED, u);
        if (ks < RKS) {
          float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll                                         // samples ks, ks + RKS, ... in order; the loads run ahead of the FMAs
          for (int i = 0; i < (RKC + RKS - 1) / RKS; ++i) {
            const int k = ks + i * RKS;
            if (k < kn) {
              const float dk = s.dh[k][jj];
              const float4 pk = s.p2[k][ii4];
              acc.x = fmaf(dk, pk.x, acc.x); acc.y = fmaf(dk, pk.y, acc.y); acc.z = fmaf(dk, pk.z, acc.z); acc.w = fmaf(dk, pk.w, acc.w);
            }
          }
          s.part[ks * RED_TILE_VEC + vec] = acc;
        }
        __syncthreads();
        if (tid < RED_TILE_VEC) {
#pragma unroll
          for (int g = 0; g < RKS; ++g) f4_add(total, s.part[g * RED_TILE_VEC + tid]);
        }
        if (k0 + RKC >= n_samples) break;
      }
      if (tid < RED_TILE_VEC) emit(v, total, held);
      if (tid == 0) at(RED_AT_EMITTED, u);
    } else {
      const int o0 = (u - RED_FC1_TILES) * RV, nv = min(RV, RED_OTHER - o0);
      const int vi = tid % RV, sg = tid / RV;
      const int o = o0 + vi, v = o < W3 / 4 ? o : o + 4000;     // skip the fc1.weight vectors
      if (tid < nv) held = pre(v);                              // (tid < nv: vi == tid, sg == 0)
      if (sg < RSS && vi < nv) {
        const float4* ps = reinterpret_cast<const float4*>(slots) + v;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        // slots sg, sg + RSS, ... in order; a batch of RSLOT_BATCH loads is in flight before the first add
        for (int s0 = sg;; s0 += RSLOT_BATCH * RSS) {
          float4 q[RSLOT_BATCH];
#pragma unroll
          for (int i = 0; i < RSLOT_BATCH; ++i)
            if (s0 + i * RSS < n_slots) q[i] = __ldcg(ps + (size_t)(s0 + i * RSS) * (DET_STRIDE / 4));
          if (s0 == sg && tid == 0) at(RED_AT_ISSUED, u);
#pragma unroll
          for (int i = 0; i < RSLOT_BATCH; ++i)
            if (s0 + i * RSS < n_slots) f4_add(acc, q[i]);
          if (s0 + RSLOT_BATCH * RSS >= n_slots) break;
        }
        s.part[sg * RV + vi] = acc;
      }
      __syncthreads();
      if (tid == 0) at(RED_AT_LOADED, u);
      if (tid < nv) {
        float4 total = s.part[tid];
#pragma unroll 5
        for (int g = 1; g < RSS; ++g) f4_add(total, s.part[g * RV + tid]);
        emit(v, total, held);
      }
      if (tid == 0) at(RED_AT_EMITTED, u);
    }
  }
}

// {sum of the slots' batch-mean nll terms, sum of their correct counts}, in slot order per lane and a fixed butterfly across
// the lanes; called by all 32 lanes of one warp, every lane gets the result.
__device__ __forceinline__ float2 reduce_loss(const float* __restrict__ slots, int n_slots) {
  const int lane = threadIdx.x & 31;
  float l = 0.f, c = 0.f;
  for (int sl = lane; sl < n_slots; sl += 32) {
    l += __ldcg(slots + (size_t)sl * DET_STRIDE + NPAR);
    c += __ldcg(slots + (size_t)sl * DET_STRIDE + NPAR + 1);
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    l += __shfl_xor_sync(0xffffffffu, l, d);
    c += __shfl_xor_sync(0xffffffffu, c, d);
  }
  return make_float2(l, c);
}

}  // namespace cn
