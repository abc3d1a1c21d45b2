// Forward-only, eval-mode pass of the tutorial's `Net` (no dropout) over N samples, for test-set evaluation: per-sample
// log-probabilities (optional), and the sums {nll, #correct, #samples} over all N samples in one deterministic result.
//
// Written for throughput rather than per-sample latency (the training step kernel, convnet.cu, carries ONE sample per CTA
// and stages all weights for it).  Here a persistent grid of at most as many CTAs as fit resident stages the weights once
// per CTA and walks over groups of S samples:
//   * weights: 1-D bulk copies of w1|b1, b2 and w3|b3|w4|b4 straight from `params`; conv2.weight is scattered once into
//     the layout conv2 reads (w2 below).  Only `params` is read, so any packed `Net` works.
//   * images: the S images of a group are one contiguous range of x, brought in by one bulk copy.  uint8 images land in
//     a staging buffer and are normalised into x with the caller's mean / std; the copy of the next group is issued as
//     soon as the staging buffer is free (after that conversion), so it overlaps the whole group.  float32 images are
//     copied into x directly, after conv1 has read the current group.
//   * fp32 SIMT throughout (no tensor cores): predictions must match the fp32 model, and bf16 operands flip near-tie
//     argmaxes.  Argmax ties go to the lowest index, like torch.argmax and the step kernel's S4.
//   * determinism: a CTA sums its samples in a fixed order (fp32 loss, integer count) into its own slot; the last CTA to
//     finish (ticket counter + fence) adds the slots in CTA order, the loss in fp64.  No float atomics, so two calls on the
//     same device and input are bit-equal.
//
// Flat parameter layout: see convnet_args.cuh (W1 .. NPAR).
#include <cstddef>
#include <cstdint>
#include <cstring>
#include "tc_common.cuh"
#include "convnet_args.cuh"

namespace ce {

using cn::B1; using cn::B2; using cn::B3; using cn::B4; using cn::NPAR; using cn::W1; using cn::W2; using cn::W3; using cn::W4;

constexpr int S = 8;           // samples in flight per CTA: conv2 has S x 16 pooled cells x 4 channel groups = T work items
constexpr int T = 512;
constexpr int P1S = 1441;      // per-sample stride of p1 [S][10][12][12]: odd, so the two samples of a conv2 warp take opposite
                               // bank parities, and with row stride 12 the 16 cells of one sample hit 16 distinct even banks
constexpr int P2S = 336;       // per-sample stride of p2 [S][320] (16-byte multiple, = 16 mod 32)
constexpr int HS = 52;         // per-sample stride of h [S][50]
constexpr int W2ROW = 32;      // conv2.weight as w2[ci*25 + k][g*8 + c] = W[co = 5g + c][ci][k]: a float4 + a float per tap
static_assert(S * 16 * 4 == T, "conv2: one (sample, pooled cell, group of 5 output channels) per thread");
static_assert(T / 8 >= 50 && S == 8, "fc1: 8 lanes per output row, lane l8 writes sample l8");

struct __align__(16) Smem {
  alignas(16) float w1[252];
  float b1[12];
  alignas(16) float b2[20];
  alignas(16) float w3[16000];   // w3 | b3 | w4 | b4 as in params (one bulk copy)
  float b3[52];
  float w4[500];
  float b4[12];
  alignas(16) float w2[250 * W2ROW];
  alignas(16) float x[S * 784];  // normalised images of the current group
  alignas(16) float p1[(S * P1S + 3) / 4 * 4];
  alignas(16) float p2[S * P2S];
  alignas(16) float h[S * HS];
  alignas(16) unsigned char raw[S * 784];   // uint8 images of the next group (bulk-copy target)
  float nll[S];
  int corr[S];
  uint64_t bar_w, bar_x;
  int is_last;
};
static_assert(offsetof(Smem, b1) == offsetof(Smem, w1) + (B1 - W1) * 4 && offsetof(Smem, b3) == offsetof(Smem, w3) + (B3 - W3) * 4 &&
                  offsetof(Smem, w4) == offsetof(Smem, w3) + (W4 - W3) * 4 && offsetof(Smem, b4) == offsetof(Smem, w3) + (B4 - W3) * 4,
              "bulk-copied weight groups must be laid out as in params");
static_assert(sizeof(Smem) <= 232448, "fits the 227 KB opt-in of one CTA");

struct EvalArgs {
  const float* params;
  const void* x;             // uint8 [N,28,28] or normalised float32 [N,1,28,28]
  const long long* target;   // [N]
  double* result;            // [3]: nll sum, #correct, #samples
  int* slots;                // [0] ticket (0 between launches), then (loss bits, #correct) per CTA
  float* out_logp;           // [N,10] or null
  long long N;
  int x_u8;
  float mean, inv_std;
};

__global__ void __launch_bounds__(T, 1) convnet_eval_kernel(EvalArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* __restrict__ P = a.params;
  const long long ngroups = (a.N + S - 1) / S;
  const unsigned int img_bytes = a.x_u8 ? 784u : 3136u;
  unsigned char* const img_dst = a.x_u8 ? s.raw : reinterpret_cast<unsigned char*>(s.x);
  auto load_group = [&](long long g) {      // one thread: the group's images as one bulk copy
    const long long b0 = g * S;
    const unsigned int n = (unsigned int)(a.N - b0 < S ? a.N - b0 : S);
    tc::mbar_expect_tx(&s.bar_x, n * img_bytes);
    tc::bulk_g2s(img_dst, reinterpret_cast<const unsigned char*>(a.x) + (size_t)b0 * img_bytes, n * img_bytes, &s.bar_x);
  };

  if (tid == 0) {
    tc::mbar_init(&s.bar_w, 1);
    tc::mbar_init(&s.bar_x, 1);
    tc::mbar_fence_init();
    tc::fence_proxy_async_global();         // params / x may have been written by the previous kernel
    tc::mbar_expect_tx(&s.bar_w, (W2 - W1) * 4 + 80 + (NPAR - W3) * 4);
    tc::bulk_g2s(s.w1, P + W1, (W2 - W1) * 4, &s.bar_w);             // w1 | b1
    tc::bulk_g2s(s.b2, P + B2, 80, &s.bar_w);
    tc::bulk_g2s(s.w3, P + W3, (NPAR - W3) * 4, &s.bar_w);           // w3 | b3 | w4 | b4
    load_group(blockIdx.x);
  }
  {
    // conv2.weight [co][ci][k] -> w2[ci*25 + k][(co/5)*8 + co%5]: all loads in flight before the first store
    const float4* __restrict__ P4w2 = reinterpret_cast<const float4*>(P + W2);
    float4 v[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int i4 = tid + k * T;
      v[k] = i4 < 1250 ? __ldg(P4w2 + i4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int i4 = tid + k * T;
      if (i4 < 1250) {
        const float w[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int i = i4 * 4 + e, co = i / 250, r = i % 250;
          s.w2[r * W2ROW + (co / 5) * 8 + co % 5] = w[e];
        }
      }
    }
  }
  float loss_local = 0.f;                   // thread 0: this CTA's samples, in order
  int correct_local = 0;
  __syncthreads();                          // mbarrier initialisation visible before any wait

  unsigned int it = 0;
  for (long long g = blockIdx.x; g < ngroups; g += gridDim.x, ++it) {
    const long long b0 = g * S;
    const int n = (int)(a.N - b0 < S ? a.N - b0 : S);
    const bool has_next = g + gridDim.x < ngroups;
    const long long y = warp < n ? __ldg(a.target + b0 + warp) : -1;   // fc2: warp w takes sample w
    tc::mbar_wait(&s.bar_x, it & 1u);       // this group's images
    if (a.x_u8) {
      for (int q = tid; q < n * 49; q += T) {          // 16 pixels per thread-iteration
        const uint4 r = *reinterpret_cast<const uint4*>(s.raw + q * 16);
        const unsigned int wv[4] = {r.x, r.y, r.z, r.w};
        float f[16];
#pragma unroll
        for (int e = 0; e < 16; ++e) f[e] = ((float)((wv[e >> 2] >> ((e & 3) * 8)) & 0xffu) * (1.f / 255.f) - a.mean) * a.inv_std;
        float4* dst = reinterpret_cast<float4*>(s.x + q * 16);
#pragma unroll
        for (int e = 0; e < 4; ++e) dst[e] = make_float4(f[4 * e], f[4 * e + 1], f[4 * e + 2], f[4 * e + 3]);
      }
      __syncthreads();                      // staging buffer consumed: the next group's copy overlaps this whole group
      if (tid == 0 && has_next) load_group(g + gridDim.x);
    }
    if (it == 0) tc::mbar_wait(&s.bar_w, 0);

    // ------------------------------------------------------------ conv1 -> maxpool2 -> relu    (p1 [S][10][12][12])
    if (tid < 480) {                        // 48 threads per channel: the 25 weights stay in registers
      const int c = tid / 48;
      float w[25];
#pragma unroll
      for (int k = 0; k < 25; ++k) w[k] = s.w1[c * 25 + k];
      const float bias = s.b1[c];
#pragma unroll 1
      for (int j = tid - c * 48; j < n * 144; j += 48) {
        const int smp = j / 144, r = j - smp * 144, py = r / 12, px = r - py * 12;
        const float* xs = s.x + smp * 784 + (2 * py) * 28 + 2 * px;
        float patch[6][6];
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
          for (int jj = 0; jj < 3; ++jj) {
            const float2 q = *reinterpret_cast<const float2*>(xs + i * 28 + 2 * jj);
            patch[i][2 * jj] = q.x; patch[i][2 * jj + 1] = q.y;
          }
        float a00 = bias, a01 = bias, a10 = bias, a11 = bias;
#pragma unroll
        for (int ky = 0; ky < 5; ++ky)
#pragma unroll
          for (int kx = 0; kx < 5; ++kx) {
            const float wk = w[ky * 5 + kx];
            a00 = fmaf(wk, patch[ky][kx], a00);
            a01 = fmaf(wk, patch[ky][kx + 1], a01);
            a10 = fmaf(wk, patch[ky + 1][kx], a10);
            a11 = fmaf(wk, patch[ky + 1][kx + 1], a11);
          }
        s.p1[smp * P1S + c * 144 + r] = fmaxf(fmaxf(fmaxf(a00, a01), fmaxf(a10, a11)), 0.f);
      }
    }
    __syncthreads();
    if (!a.x_u8 && tid == 0 && has_next) load_group(g + gridDim.x);   // x consumed: the next float32 group lands in it

    // ------------------------------------------------------------ conv2 -> maxpool2 -> relu    (p2 [S][320])
    {
      // warps 4g .. 4g+3 take output channels 5g .. 5g+4 (weight loads are warp-wide broadcasts); lane = (sample, cell)
      const int grp = warp >> 2, smp = (warp & 3) * 2 + (lane >> 4), cell = lane & 15, py = cell >> 2, px = cell & 3;
      if (smp < n) {
        float acc[4][5];
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
          for (int c = 0; c < 5; ++c) acc[p][c] = 0.f;
        const float* src = s.p1 + smp * P1S + (2 * py) * 12 + 2 * px;
#pragma unroll 1
        for (int ci = 0; ci < 10; ++ci) {
          float patch[6][6];
#pragma unroll
          for (int i = 0; i < 6; ++i)
#pragma unroll
            for (int j = 0; j < 6; ++j) patch[i][j] = src[ci * 144 + i * 12 + j];
          const float* wrow = s.w2 + ci * 25 * W2ROW + grp * 8;
#pragma unroll
          for (int ky = 0; ky < 5; ++ky)
#pragma unroll
            for (int kx = 0; kx < 5; ++kx) {
              const float* wp = wrow + (ky * 5 + kx) * W2ROW;
              const float4 w = *reinterpret_cast<const float4*>(wp);
              const float wl[5] = {w.x, w.y, w.z, w.w, wp[4]};
              const float in[4] = {patch[ky][kx], patch[ky][kx + 1], patch[ky + 1][kx], patch[ky + 1][kx + 1]};
#pragma unroll
              for (int p = 0; p < 4; ++p)
#pragma unroll
                for (int c = 0; c < 5; ++c) acc[p][c] = fmaf(wl[c], in[p], acc[p][c]);
            }
        }
#pragma unroll
        for (int c = 0; c < 5; ++c) {
          const int co = grp * 5 + c;
          const float bias = s.b2[co];
          const float m = fmaxf(fmaxf(acc[0][c] + bias, acc[1][c] + bias), fmaxf(acc[2][c] + bias, acc[3][c] + bias));
          s.p2[smp * P2S + co * 16 + cell] = fmaxf(m, 0.f);
        }
      }
    }
    __syncthreads();

    // ------------------------------------------------------------ fc1 + relu: [S x 320] x [320 x 50]
    {
      // 8 lanes per output row j, 40 inputs each; every fc1.weight float4 read from shared memory feeds 4 x S FMAs
      const int j = tid >> 3, l8 = tid & 7;
      float acc[S];
#pragma unroll
      for (int q = 0; q < S; ++q) acc[q] = 0.f;
      if (j < 50) {
        const float4* wrow = reinterpret_cast<const float4*>(s.w3 + j * 320);
#pragma unroll 2
        for (int k = 0; k < 10; ++k) {
          const float4 w = wrow[l8 + 8 * k];
#pragma unroll
          for (int q = 0; q < S; ++q) {
            const float4 v = *reinterpret_cast<const float4*>(s.p2 + q * P2S + (l8 + 8 * k) * 4);
            acc[q] = fmaf(w.x, v.x, acc[q]); acc[q] = fmaf(w.y, v.y, acc[q]);
            acc[q] = fmaf(w.z, v.z, acc[q]); acc[q] = fmaf(w.w, v.w, acc[q]);
          }
        }
      }
      float mine = 0.f;
#pragma unroll
      for (int q = 0; q < S; ++q) {
        float v = acc[q];
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        if (l8 == q) mine = v;
      }
      if (j < 50) s.h[l8 * HS + j] = fmaxf(mine + s.b3[j], 0.f);   // lane l8 of the row writes sample l8
    }
    __syncthreads();

    // ------------------------------------------------------------ fc2 + log_softmax + nll + argmax: warp w, sample w
    if (warp < n) {
      float logit = -INFINITY;
      if (lane < 10) {
        float acc = s.b4[lane];
        const float* hv = s.h + warp * HS;
#pragma unroll 10
        for (int i = 0; i < 50; ++i) acc = fmaf(s.w4[lane * 50 + i], hv[i], acc);
        logit = acc;
      }
      float mx = logit; int am = lane;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        const float o = __shfl_xor_sync(0xffffffffu, mx, d);
        const int oi = __shfl_xor_sync(0xffffffffu, am, d);
        if (o > mx || (o == mx && oi < am)) { mx = o; am = oi; }
      }
      float se = lane < 10 ? __expf(logit - mx) : 0.f;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) se += __shfl_xor_sync(0xffffffffu, se, d);
      const float logp = logit - (mx + __logf(se));   // -inf on lanes >= 10
      if (lane < 10 && a.out_logp != nullptr) a.out_logp[(size_t)(b0 + warp) * 10 + lane] = logp;
      // a label outside [0, 10) reads lane 10's -inf: the loss sum becomes +inf instead of silently wrong
      const float ly = __shfl_sync(0xffffffffu, logp, (y >= 0 && y < 10) ? (int)y : 10);
      if (lane == 0) { s.nll[warp] = -ly; s.corr[warp] = am == y ? 1 : 0; }
    }
    __syncthreads();
    if (tid == 0)
      for (int w = 0; w < n; ++w) { loss_local += s.nll[w]; correct_local += s.corr[w]; }
  }

  // ---------------------------------------------------------------- per-CTA slot, then the last CTA adds them in CTA order
  if (tid == 0) {
    a.slots[1 + 2 * blockIdx.x] = __float_as_int(loss_local);
    a.slots[2 + 2 * blockIdx.x] = correct_local;
    __threadfence();
    const unsigned int ticket = atomicAdd(reinterpret_cast<unsigned int*>(a.slots), 1u);
    s.is_last = ticket == gridDim.x - 1;
  }
  __syncthreads();
  if (s.is_last && tid == 0) {
    __threadfence();
    double loss = 0.0;
    long long correct = 0;
    for (unsigned int c = 0; c < gridDim.x; ++c) {
      loss += (double)__int_as_float(__ldcg(a.slots + 1 + 2 * c));
      correct += __ldcg(a.slots + 2 + 2 * c);
    }
    a.result[0] = loss;
    a.result[1] = (double)correct;
    a.result[2] = (double)a.N;
    a.slots[0] = 0;                         // ready for the next launch on this slot buffer
  }
}

}  // namespace ce

extern "C" {

// Resident CTAs of the eval kernel on `dev` (0 on error): its grid never exceeds this, and the slot buffer holds 2 + 2 x this.
int b2_convnet_eval_max_ctas(int dev) {
  static int cached[64] = {0};
  if (dev < 0 || dev >= 64) return 0;
  if (cached[dev] == 0) {
    const int smem = (int)sizeof(ce::Smem);
    if (cudaFuncSetAttribute(ce::convnet_eval_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return 0;
    int per_sm = 0, sms = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ce::convnet_eval_kernel, ce::T, smem) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    cached[dev] = per_sm * sms;
  }
  return cached[dev];
}

int b2_convnet_eval_samples_per_cta() { return ce::S; }

// N == 0: nothing is launched; result is zeroed.
int b2_convnet_eval_launch(const float* params, const void* x, int x_u8, const long long* target, double* result, int* slots,
                           float* out_logp, long long N, float mean, float std, int dev, cudaStream_t stream) {
  if (N <= 0) return (int)cudaMemsetAsync(result, 0, 3 * sizeof(double), stream);
  const int max_ctas = b2_convnet_eval_max_ctas(dev);
  if (max_ctas <= 0) return (int)cudaErrorInvalidConfiguration;
  const long long groups = (N + ce::S - 1) / ce::S;
  const int grid = groups < max_ctas ? (int)groups : max_ctas;
  ce::EvalArgs a;
  a.params = params; a.x = x; a.target = target; a.result = result; a.slots = slots; a.out_logp = out_logp;
  a.N = N; a.x_u8 = x_u8; a.mean = mean; a.inv_std = 1.f / std;
  ce::convnet_eval_kernel<<<grid, ce::T, sizeof(ce::Smem), stream>>>(a);
  return (int)cudaGetLastError();
}

}  // extern "C"
