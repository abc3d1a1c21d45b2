// Batched (large per-GPU batch) training engine for the tutorial ConvNet on sm_90a: layer-wise kernels over the whole
// batch, with the GEMM-shaped layers on the Hopper tensor cores (wgmma.mma_async, accumulators in registers) fed by TMA.
//
// The per-sample fused kernels (convnet.cu / convnet_cluster.cu) are built for the reference's latency-bound configuration
// (global batch 128, train_dist.py:85).  At B >= 1024 per GPU the same network is throughput-bound, and 66 % of its MACs
// are the three conv2 GEMMs (train_dist.py:59,66 and their backward), so here:
//
//   conv1 -> pool -> relu             bt_conv1_fwd     SIMT (K = 25: not GEMM-shaped); writes P1 as bf16 NHWC [B,12,12,16]
//   conv2 -> dropout2d -> pool -> relu bt_conv2_fwd    wgmma: implicit GEMM, M = 128 rows = 2 samples x 64 positions,
//                                                       N = 32 (20 channels), K = 25 taps x 16 input channels.  TMA IS the
//                                                       im2col: one 4-D box {16 c, 8 x, 8 y, 2 b} per tap at offset (kx, ky)
//                                                       lands as a K-major 32B-swizzled A tile (one 32-byte row per output
//                                                       position); bias/dropout2d/pool/relu run in the register epilogue.
//                                                       (Channel-last because TMA needs a 16-byte aligned innermost start:
//                                                       an x-innermost box shifted by kx elements is not a legal box start.)
//   fc1 (+bias, relu)                  gemm_tcgen05.cu  the library GEMM of this repo (TMA + wgmma), N = 64
//   dropout, fc2, log_softmax, nll,    bt_head          SIMT, one thread per sample (2 kFLOP/sample)
//   and their backward down to dH
//   fc1 data gradient                  gemm_tcgen05.cu  dP2 = dH x W3
//   pool/relu/dropout2d backward       bt_route         dP2 -> dC (bf16, NCHW [B,32,8,8])
//   conv2 weight (+bias) gradient      bt_conv2_wgrad   wgmma: D[(tap,ci), co] = sum over positions; the same 25 TMA tap
//                                                       boxes per sample are now the MN-major A operand (M = 8 taps x 16
//                                                       channels per instruction), dC the K-major B operand; the bias
//                                                       gradient falls out of a constant-one input channel.
//   conv2 data gradient                bt_conv2_dgrad   wgmma: dA[pos, (tap,ci)] = dC x W2 (N = 400 as 5 x 80), then
//                                                       col2im + relu/pool routing of conv1 in the epilogue
//   conv1 weight gradient              bt_conv1_wgrad   SIMT (sparse: one of four positions per pooled cell)
//   fc weight/bias gradients           bt_fc_wgrad      SIMT register tiles
//   bf16 operand copies of the weights bt_pack_weights  after every optimizer step
//
// Gradients are accumulated with red.add into the same flat fp32 bucket layout as the per-sample engine (convnet_args.cuh),
// so the fused all-reduce + SGD kernel (sgd.cu) is shared.  Activations between kernels are bf16 and stay L2-resident
// (< 20 KB per sample).  Dropout masks come from the same Philox stream as the per-sample engine, so both engines can be
// compared with identical masks.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

#include "common.cuh"
#include "tc_common.cuh"
#include "convnet_args.cuh"

namespace bt {

using cn::W1; using cn::B1; using cn::W2; using cn::B2; using cn::W3; using cn::B3; using cn::W4; using cn::B4;

constexpr int P1_SAMPLE = 12 * 12 * 16;       // bf16 elements per sample of P1 [12 y][12 x][16 c] (channels 10..15: 1, 0, 0, 0, 0, 0)
constexpr int DC_SAMPLE = 32 * 64;            // bf16 elements per sample of dC [32 co][64 pos]
constexpr int W2K_K = 448;                    // 28 taps x 16 channels (25 real taps)
constexpr int W2R_N = 400;                    // 25 taps x 16 channels

struct Common {
  unsigned long long seed;
  const unsigned long long* step;   // device step counter (RNG offset), may be null
  long long sample_base;
  int B;
  int training;
  float p_drop;
};

__device__ __forceinline__ float drop_scale(float u, float p, float keep, int training) {
  return training ? (u >= p ? keep : 0.f) : 1.f;
}
__device__ __forceinline__ unsigned short bf16_bits(float v) {
  __nv_bfloat16 h = __float2bfloat16(v);
  return *reinterpret_cast<unsigned short*>(&h);
}
__device__ __forceinline__ float bf16_to_f32(unsigned short b) { return __uint_as_float((uint32_t)b << 16); }

// =====================================================================================================================
// conv1 (1->10, 5x5) + maxpool2 + relu.  288 threads = 2 samples x 144 pooled positions; a thread computes all 10 channels
// of its position from one 6x6 input patch held in registers (1000 FMA per 18 shared-memory loads).
// =====================================================================================================================
__global__ void __launch_bounds__(288) bt_conv1_fwd(const float* __restrict__ params, const void* __restrict__ x, int x_u8,
                                                    float mean, float inv_std, int B, __nv_bfloat16* __restrict__ P1,
                                                    unsigned char* __restrict__ A1) {
  __shared__ __align__(16) float xs[2][28 * 28];
  __shared__ __align__(16) float w1s[10][28];                       // 25 weights + bias + pad
  const int tid = threadIdx.x;
  for (int i = tid; i < 280; i += 288) {
    const int c = i / 28, k = i % 28;
    w1s[c][k] = k < 25 ? params[W1 + c * 25 + k] : (k == 25 ? params[B1 + c] : 0.f);
  }
  const int sl = tid / 144, pos = tid % 144, py = pos / 12, px = pos % 12;
  for (int pair = blockIdx.x; pair * 2 < B; pair += gridDim.x) {
    const int b0 = pair * 2;
    __syncthreads();                                                // previous iteration is done with xs
    if (x_u8) {
      for (int i = tid; i < 98; i += 288) {                         // 2 x 49 uint4
        const int s = i / 49, q = i % 49;
        if (b0 + s < B) {
          const uint4 v = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const unsigned char*>(x) + (size_t)(b0 + s) * 784) + q);
          const unsigned int wv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int e = 0; e < 16; ++e)
            xs[s][q * 16 + e] = ((float)((wv[e >> 2] >> ((e & 3) * 8)) & 0xffu) * (1.f / 255.f) - mean) * inv_std;
        }
      }
    } else {
      for (int i = tid; i < 392; i += 288) {                        // 2 x 196 float4
        const int s = i / 196, q = i % 196;
        if (b0 + s < B)
          reinterpret_cast<float4*>(xs[s])[q] = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(x) + (size_t)(b0 + s) * 784) + q);
      }
    }
    __syncthreads();
    if (b0 + sl < B) {
      float patch[6][6];
#pragma unroll
      for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          const float2 q = *reinterpret_cast<const float2*>(&xs[sl][(2 * py + i) * 28 + 2 * px + 2 * j]);
          patch[i][2 * j] = q.x; patch[i][2 * j + 1] = q.y;
        }
      float outv[10];
      unsigned char* a1 = A1 + (size_t)(b0 + sl) * 1440 + pos;
#pragma unroll
      for (int c = 0; c < 10; ++c) {
        float w[28];
#pragma unroll
        for (int k4 = 0; k4 < 7; ++k4) {
          const float4 q = *reinterpret_cast<const float4*>(&w1s[c][k4 * 4]);
          w[k4 * 4] = q.x; w[k4 * 4 + 1] = q.y; w[k4 * 4 + 2] = q.z; w[k4 * 4 + 3] = q.w;
        }
        float a00 = w[25], a01 = w[25], a10 = w[25], a11 = w[25];
#pragma unroll
        for (int ky = 0; ky < 5; ++ky)
#pragma unroll
          for (int kx = 0; kx < 5; ++kx) {
            const float ww = w[ky * 5 + kx];
            a00 = fmaf(ww, patch[ky][kx], a00);
            a01 = fmaf(ww, patch[ky][kx + 1], a01);
            a10 = fmaf(ww, patch[ky + 1][kx], a10);
            a11 = fmaf(ww, patch[ky + 1][kx + 1], a11);
          }
        float m = a00; int arg = 0;
        if (a01 > m) { m = a01; arg = 1; }
        if (a10 > m) { m = a10; arg = 2; }
        if (a11 > m) { m = a11; arg = 3; }
        outv[c] = fmaxf(m, 0.f);
        a1[c * 144] = (unsigned char)(arg | (m > 0.f ? 0 : 4));     // consecutive threads -> consecutive bytes
      }
      // one 32-byte NHWC pixel: 10 channels, the constant-one channel (conv2 bias-gradient row), 5 zero channels
      uint4* dst = reinterpret_cast<uint4*>(P1 + (size_t)(b0 + sl) * P1_SAMPLE + pos * 16);
      dst[0] = make_uint4(b2::pack_bf16x2(outv[0], outv[1]), b2::pack_bf16x2(outv[2], outv[3]), b2::pack_bf16x2(outv[4], outv[5]),
                          b2::pack_bf16x2(outv[6], outv[7]));
      dst[1] = make_uint4(b2::pack_bf16x2(outv[8], outv[9]), b2::pack_bf16x2(1.f, 0.f), 0u, 0u);
    }
  }
}

// =====================================================================================================================
// conv2 forward on wgmma: implicit GEMM with TMA as the im2col engine.
// =====================================================================================================================
// One TMA box per tile brings the whole 12x12x16 input of TWO samples into shared memory as [y][b][x][c] (32-byte pixels,
// 32B swizzle); the 25 filter taps are then 25 shared-memory DESCRIPTORS over that image -- start address shifted by
// (ky*768 + kx*32) bytes, 8-row groups (one output row of one sample) 384 bytes apart -- so the im2col costs no data movement
// at all (the first version issued one TMA box per tap: 25x the L2->SM traffic, 70 us at B = 4096).  Accumulator row
// r = (oy*2 + b)*8 + ox.  Descriptor arithmetic checked on hardware by tests/test_gpu_tc_probe.py.
constexpr int C2F_NST = 4;
constexpr int C2F_IMG = 12 * 2 * 12 * 32;     // 9216 B
constexpr int BT_THREADS = 384;               // warpgroup 0: TMA producer, warpgroups 1, 2: wgmma + epilogue (64 rows each)
struct __align__(1024) C2fSmem {
  uint8_t w[7][4096];                 // W2 as B operand: 7 K-blocks of [32 co rows x 64 k], k = (tap % 4) * 16 + ci
  uint8_t a[C2F_NST][C2F_IMG];        // [12 y][2 b][12 x][16 c] bf16
  float stage[128][21];
  float m2[2][20];
  float bias[20];
  uint64_t full[C2F_NST], empty[C2F_NST], wfull;
};

__global__ void __launch_bounds__(BT_THREADS, 1)
bt_conv2_fwd(const __grid_constant__ CUtensorMap map_p1, const __grid_constant__ CUtensorMap map_w2k,
             const float* __restrict__ params, Common cm, __nv_bfloat16* __restrict__ P2, unsigned char* __restrict__ A2) {
  extern __shared__ uint8_t smem_raw[];
  C2fSmem& s = *reinterpret_cast<C2fSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int tiles = (cm.B + 1) / 2;
  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&map_p1); tc::prefetch_tmap(&map_w2k);
    for (int i = 0; i < C2F_NST; ++i) { tc::mbar_init(&s.full[i], 1); tc::mbar_init(&s.empty[i], 256); }
    tc::mbar_init(&s.wfull, 1);
    tc::mbar_fence_init();
  }
  if (threadIdx.x < 20) s.bias[threadIdx.x] = params[B2 + threadIdx.x];
  __syncthreads();

  if (wg == 0) {
    // ======================================================== TMA producer: one box per tile
    if (t == 0) {
      tc::mbar_expect_tx(&s.wfull, 7 * 4096);
      for (int j = 0; j < 7; ++j) tc::tma_load_2d(s.w[j], &map_w2k, &s.wfull, j * 64, 0);
      uint32_t it = 0;
      for (int tt = blockIdx.x; tt < tiles; tt += gridDim.x, ++it) {
        const int st = it % C2F_NST;
        tc::mbar_wait(&s.empty[st], ((it / C2F_NST) & 1) ^ 1);
        tc::mbar_expect_tx(&s.full[st], C2F_IMG);
        tc::tma_load_4d(s.a[st], &map_p1, &s.full[st], 0, 0, 2 * tt, 0);      // dims (c, x, b, y)
      }
    }
    return;
  }
  // ========================================================== 25 taps = 25 descriptors over the image, then bias,
  // dropout2d, 2x2 max-pool, relu.  Warpgroup h owns accumulator rows 64h..64h+63 = row groups (oy*2 + b) 8h..8h+7.
  const int h = wg - 1, e = threadIdx.x - 128;
  const float keep = 1.f / (1.f - cm.p_drop);
  const unsigned long long step = cm.step ? *cm.step : 0ull;
  tc::mbar_wait(&s.wfull, 0);
  uint32_t it = 0;
  for (int tt = blockIdx.x; tt < tiles; tt += gridDim.x, ++it) {
    const int st = it % C2F_NST;
    const int b0 = 2 * tt;
    if (e < 10) {
      const int sb = e / 5, qq = e % 5;
      const uint4 rr = b2::Philox::gen(cm.seed, (unsigned long long)(cm.sample_base + b0 + sb), step * 32ull + qq);
      const float k = 2.3283064365386963e-10f;
      s.m2[sb][qq * 4 + 0] = drop_scale(rr.x * k, cm.p_drop, keep, cm.training);
      s.m2[sb][qq * 4 + 1] = drop_scale(rr.y * k, cm.p_drop, keep, cm.training);
      s.m2[sb][qq * 4 + 2] = drop_scale(rr.z * k, cm.p_drop, keep, cm.training);
      s.m2[sb][qq * 4 + 3] = drop_scale(rr.w * k, cm.p_drop, keep, cm.training);
    }
    tc::mbar_wait(&s.full[st], (it / C2F_NST) & 1);
    float d[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) d[i] = 0.f;
    const uint32_t img = tc::smem_u32(s.a[st]) + h * 8 * 384;
    tc::wg_fence();
#pragma unroll
    for (int tap = 0; tap < 25; ++tap) {
      const int ky = tap / 5, kx = tap - ky * 5;
      const uint64_t ad = tc::smem_desc(img + ky * 768 + kx * 32, 16, /*SBO: next (oy, b) row group*/ 384, tc::kSw32);
      const uint64_t bd = tc::smem_desc(tc::smem_u32(s.w[tap >> 2]) + (tap & 3) * 32, 16, 1024, tc::kSw128);
      tc::mma<32>(d, ad, bd, tap > 0 ? 1u : 0u);
    }
    tc::wg_commit();
    tc::wg_wait_all();
    tc::acc_fence<16>(d);
    tc::mbar_arrive(&s.empty[st]);                              // image consumed: the producer may refill the stage
    tc::named_bar_sync(1, 256);                                 // m2 visible; the previous tile's pooling is done
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int r = h * 64 + tc::acc_row(t, i), co = tc::acc_col(t, i);   // accumulator row = (oy*2 + b)*8 + ox
      const int bl = (r >> 3) & 1, srow = bl * 64 + (r >> 4) * 8 + (r & 7); // staging row = b*64 + oy*8 + ox
      if (co < 20) s.stage[srow][co] = (d[i] + s.bias[co]) * s.m2[bl][co];
    }
    tc::named_bar_sync(1, 256);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const int o = e + 256 * i;
      if (o >= 640) break;
      const int sb = o / 320, oo = o % 320, co = oo >> 4, cell = oo & 15;
      const int p00 = sb * 64 + (2 * (cell >> 2)) * 8 + 2 * (cell & 3);
      const float v0 = s.stage[p00][co], v1 = s.stage[p00 + 1][co], v2 = s.stage[p00 + 8][co], v3 = s.stage[p00 + 9][co];
      float m = v0; int arg = 0;
      if (v1 > m) { m = v1; arg = 1; }
      if (v2 > m) { m = v2; arg = 2; }
      if (v3 > m) { m = v3; arg = 3; }
      if (b0 + sb < cm.B) {
        P2[(size_t)(b0 + sb) * 320 + oo] = __float2bfloat16(fmaxf(m, 0.f));
        A2[(size_t)(b0 + sb) * 320 + oo] = (unsigned char)(arg | (m > 0.f ? 0 : 4));
      }
    }
  }
}

// =====================================================================================================================
// head: dropout(relu(fc1)) -> fc2 -> log_softmax -> nll, and the backward of all of it down to dH.  One thread per sample.
// Hrelu [B,64] fp32 = relu(fc1 + b3) comes from the wgmma GEMM.
// =====================================================================================================================
__global__ void __launch_bounds__(128) bt_head(const float* __restrict__ params, const float* __restrict__ Hrelu,
                                               const long long* __restrict__ target, Common cm, int backward, float inv_bsz,
                                               __nv_bfloat16* __restrict__ H, __nv_bfloat16* __restrict__ DH,
                                               float* __restrict__ DLOG, float* __restrict__ loss_acc, float* __restrict__ out_logp) {
  __shared__ __align__(16) float w4s[10][52];
  __shared__ float b4s[10];
  __shared__ float lg[10][128];                    // per-thread logits, then dlogits (column = thread: conflict-free)
  __shared__ float red[2][4];
  for (int i = threadIdx.x; i < 520; i += 128) w4s[i / 52][i % 52] = (i % 52) < 50 ? params[W4 + (i / 52) * 50 + (i % 52)] : 0.f;
  if (threadIdx.x < 10) b4s[threadIdx.x] = params[B4 + threadIdx.x];
  __syncthreads();
  const int tid = threadIdx.x, b = blockIdx.x * 128 + tid;
  const float keep = 1.f / (1.f - cm.p_drop);
  const unsigned long long step = cm.step ? *cm.step : 0ull;
  float nll = 0.f, corr = 0.f;
  if (b < cm.B) {
    float h[52];
    {
      const float4* src = reinterpret_cast<const float4*>(Hrelu + (size_t)b * 64);
#pragma unroll
      for (int i = 0; i < 13; ++i) {
        const float4 q = __ldg(src + i);
        h[4 * i] = q.x; h[4 * i + 1] = q.y; h[4 * i + 2] = q.z; h[4 * i + 3] = q.w;
      }
      h[50] = 0.f; h[51] = 0.f;
    }
    // dropout: uniforms rnd[20 + j] of this sample's Philox stream (the stream of the per-sample engine, convnet.cu)
#pragma unroll
    for (int qq = 5; qq < 18; ++qq) {
      const uint4 rr = b2::Philox::gen(cm.seed, (unsigned long long)(cm.sample_base + b), step * 32ull + qq);
      const float k = 2.3283064365386963e-10f;
      const float u[4] = {rr.x * k, rr.y * k, rr.z * k, rr.w * k};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int j = qq * 4 + i - 20;
        if (j >= 0 && j < 50) h[j] *= drop_scale(u[i], cm.p_drop, keep, cm.training);
      }
    }
    float mx = -INFINITY;
    int am = 0;
#pragma unroll 1
    for (int k = 0; k < 10; ++k) {
      float a = b4s[k];
#pragma unroll
      for (int j4 = 0; j4 < 13; ++j4) {
        const float4 w = *reinterpret_cast<const float4*>(&w4s[k][j4 * 4]);
        a = fmaf(w.x, h[j4 * 4], a); a = fmaf(w.y, h[j4 * 4 + 1], a); a = fmaf(w.z, h[j4 * 4 + 2], a); a = fmaf(w.w, h[j4 * 4 + 3], a);
      }
      lg[k][tid] = a;
      if (a > mx) { mx = a; am = k; }
    }
    float se = 0.f;
#pragma unroll 1
    for (int k = 0; k < 10; ++k) se += __expf(lg[k][tid] - mx);
    const float lse = mx + __logf(se);
    const int y = (int)target[b];
#pragma unroll 1
    for (int k = 0; k < 10; ++k) {
      const float lp = lg[k][tid] - lse;
      if (out_logp) out_logp[(size_t)b * 10 + k] = lp;
      if (k == y) nll = -lp;
      lg[k][tid] = (__expf(lp) - (k == y ? 1.f : 0.f)) * inv_bsz;       // dlogit
    }
    corr = am == y ? 1.f : 0.f;
    if (backward) {
      float dh[56];
#pragma unroll
      for (int j = 0; j < 56; ++j) dh[j] = 0.f;
#pragma unroll 1
      for (int k = 0; k < 10; ++k) {
        const float dl = lg[k][tid];
#pragma unroll
        for (int j4 = 0; j4 < 13; ++j4) {
          const float4 w = *reinterpret_cast<const float4*>(&w4s[k][j4 * 4]);
          dh[j4 * 4] = fmaf(w.x, dl, dh[j4 * 4]); dh[j4 * 4 + 1] = fmaf(w.y, dl, dh[j4 * 4 + 1]);
          dh[j4 * 4 + 2] = fmaf(w.z, dl, dh[j4 * 4 + 2]); dh[j4 * 4 + 3] = fmaf(w.w, dl, dh[j4 * 4 + 3]);
        }
      }
      // relu' * dropout scale: h = relu(pre) * dm is positive exactly where both factors are
      const float sc = cm.training ? keep : 1.f;
#pragma unroll
      for (int j = 0; j < 52; ++j) dh[j] = h[j] > 0.f ? dh[j] * sc : 0.f;
      uint4* hd = reinterpret_cast<uint4*>(H + (size_t)b * 64);
      uint4* dd = reinterpret_cast<uint4*>(DH + (size_t)b * 64);
#pragma unroll
      for (int g = 0; g < 7; ++g) {
        float hv[8], dv[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          hv[i] = (g * 8 + i) < 52 ? h[(g * 8 + i) < 52 ? g * 8 + i : 0] : 0.f;
          dv[i] = dh[g * 8 + i];
        }
        hd[g] = make_uint4(b2::pack_bf16x2(hv[0], hv[1]), b2::pack_bf16x2(hv[2], hv[3]), b2::pack_bf16x2(hv[4], hv[5]), b2::pack_bf16x2(hv[6], hv[7]));
        dd[g] = make_uint4(b2::pack_bf16x2(dv[0], dv[1]), b2::pack_bf16x2(dv[2], dv[3]), b2::pack_bf16x2(dv[4], dv[5]), b2::pack_bf16x2(dv[6], dv[7]));
      }
      hd[7] = make_uint4(0u, 0u, 0u, 0u);
      dd[7] = make_uint4(0u, 0u, 0u, 0u);
      float4* dl4 = reinterpret_cast<float4*>(DLOG + (size_t)b * 16);
      dl4[0] = make_float4(lg[0][tid], lg[1][tid], lg[2][tid], lg[3][tid]);
      dl4[1] = make_float4(lg[4][tid], lg[5][tid], lg[6][tid], lg[7][tid]);
      dl4[2] = make_float4(lg[8][tid], lg[9][tid], 0.f, 0.f);
      dl4[3] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  if (loss_acc != nullptr) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) { nll += __shfl_xor_sync(0xffffffffu, nll, d); corr += __shfl_xor_sync(0xffffffffu, corr, d); }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = nll; red[1][threadIdx.x >> 5] = corr; }
    __syncthreads();
    if (threadIdx.x == 0) {
      atomicAdd(loss_acc, (red[0][0] + red[0][1] + red[0][2] + red[0][3]) * inv_bsz);
      atomicAdd(loss_acc + 1, red[1][0] + red[1][1] + red[1][2] + red[1][3]);
    }
  }
}

// =====================================================================================================================
// route: dP2 [B,320] (bf16, from the fc1 data-gradient GEMM) through relu / max-pool / dropout2d of conv2 -> dC [B,32,8,8].
// One thread per (sample, channel): 16 pooled cells -> one 128-byte row of 64 positions.
// =====================================================================================================================
__global__ void __launch_bounds__(256) bt_route(const __nv_bfloat16* __restrict__ dP2, const unsigned char* __restrict__ A2,
                                                int B, float scale, __nv_bfloat16* __restrict__ DC) {
  const int t = blockIdx.x * 256 + threadIdx.x;
  if (t >= B * 20) return;
  const int b = t / 20, co = t % 20;
  const uint4* gp = reinterpret_cast<const uint4*>(dP2 + (size_t)b * 320 + co * 16);
  const uint4 g0 = __ldg(gp), g1 = __ldg(gp + 1);
  const uint4 ac = __ldg(reinterpret_cast<const uint4*>(A2 + (size_t)b * 320 + co * 16));
  const uint32_t gw[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
  const uint32_t aw[4] = {ac.x, ac.y, ac.z, ac.w};
  uint32_t row[32];                                   // 64 bf16: word index = y * 4 + x / 2
#pragma unroll
  for (int cell = 0; cell < 16; ++cell) {
    const uint32_t gb = (gw[cell >> 1] >> ((cell & 1) * 16)) & 0xffffu;
    const uint32_t code = (aw[cell >> 2] >> ((cell & 3) * 8)) & 0xffu;
    const float g = (code & 4u) ? 0.f : bf16_to_f32((unsigned short)gb) * scale;
    const uint32_t gq = (uint32_t)bf16_bits(g);
    const int cy = cell >> 2, cx = cell & 3;
    row[(2 * cy) * 4 + cx] = (code == 0u ? gq : 0u) | ((code == 1u ? gq : 0u) << 16);
    row[(2 * cy + 1) * 4 + cx] = (code == 2u ? gq : 0u) | ((code == 3u ? gq : 0u) << 16);
  }
  uint4* dst = reinterpret_cast<uint4*>(DC + (size_t)b * DC_SAMPLE + co * 64);
#pragma unroll
  for (int i = 0; i < 8; ++i) dst[i] = make_uint4(row[4 * i], row[4 * i + 1], row[4 * i + 2], row[4 * i + 3]);
}

// =====================================================================================================================
// conv2 weight gradient on wgmma:  D[(tap, ci), co] = sum_{b, pos} P1[b, ci, oy+ky, ox+kx] * dC[b, co, pos]
// K = the 64 output positions of one sample.  A: the 25 TMA tap boxes [64 pos][16 ci] (32-byte rows, 32B swizzle) read
// MN-major, atoms of 16 channels LBO apart.  B: the 32 channel rows of
// dC, K-major.  Input channel 10 of P1 is a constant 1 => row (tap 0, ci 10) is the bias gradient.
// =====================================================================================================================
// One TMA box per sample brings its 12x12x16 input into shared memory as [y][x][c]; for each kernel row ky ONE instruction
// covers the kernel columns kx = 0..7 x 16 channels as 8 MN-major atoms 32 bytes apart (atoms 5..7 read the pixels to the
// right of the window: finite values whose output rows are never read), K = 16 output positions = two rows of the image.
// 5 accumulators (one per ky) of [128 x 32], split over two warpgroups.  Checked by tests/test_gpu_tc_probe.py.
constexpr int WG_NST = 8;
constexpr int WG_IMG = 5120;                          // 4608-byte image + padding the out-of-window atoms may read
constexpr int WG_STAGE = WG_IMG + 4096;               // + dC [32 co][64 pos]
struct __align__(1024) WgSmem {
  uint8_t st[WG_NST][WG_STAGE];
  uint64_t full[WG_NST], empty[WG_NST];
};

__global__ void __launch_bounds__(BT_THREADS, 1)
bt_conv2_wgrad(const __grid_constant__ CUtensorMap map_p1, const __grid_constant__ CUtensorMap map_dc, int B,
               float* __restrict__ grads) {
  extern __shared__ uint8_t smem_raw[];
  WgSmem& s = *reinterpret_cast<WgSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  for (int stg = 0; stg < WG_NST; ++stg)               // padding behind each image: finite (zero) forever
    for (int i = threadIdx.x; i < (WG_IMG - 4608) / 16; i += BT_THREADS)
      reinterpret_cast<uint4*>(s.st[stg] + 4608)[i] = make_uint4(0u, 0u, 0u, 0u);
  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&map_p1); tc::prefetch_tmap(&map_dc);
    for (int i = 0; i < WG_NST; ++i) { tc::mbar_init(&s.full[i], 1); tc::mbar_init(&s.empty[i], 256); }
    tc::mbar_fence_init();
  }
  tc::fence_proxy_async();
  __syncthreads();

  if (wg == 0) {
    if (t == 0) {
      uint32_t it = 0;
      for (int b = blockIdx.x; b < B; b += gridDim.x, ++it) {
        const int st = it % WG_NST;
        tc::mbar_wait(&s.empty[st], ((it / WG_NST) & 1) ^ 1);
        tc::mbar_expect_tx(&s.full[st], 4608 + 4096);
        tc::tma_load_4d(s.st[st], &map_p1, &s.full[st], 0, 0, 0, b);                  // dims (c, x, y, b): the whole image
        tc::tma_load_2d(s.st[st] + WG_IMG, &map_dc, &s.full[st], 0, 32 * b);
      }
    }
    return;
  }
  // warpgroup h: accumulator rows 64h.. = kernel columns kx = 4h..4h+3 (atoms 32 bytes apart: start + 4h * 32)
  const int h = wg - 1;
  float acc[5][16];
#pragma unroll
  for (int ky = 0; ky < 5; ++ky)
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[ky][i] = 0.f;
  uint32_t it = 0;
  for (int b = blockIdx.x; b < B; b += gridDim.x, ++it) {
    const int st = it % WG_NST;
    tc::mbar_wait(&s.full[st], (it / WG_NST) & 1);
    const uint32_t img = tc::smem_u32(s.st[st]), d0 = img + WG_IMG;
    tc::wg_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint64_t bd = tc::smem_desc(d0 + ks * 32, 16, 1024, tc::kSw128);
#pragma unroll
      for (int ky = 0; ky < 5; ++ky)
        tc::mma<32>(acc[ky], tc::smem_desc(img + h * 128 + ky * 384 + ks * 768, /*LBO: next kx*/ 32, /*SBO: next image row*/ 384, tc::kSw32),
                    bd, 1u, /*A MN-major*/ 1u);
    }
    tc::wg_commit();
    tc::wg_wait_all();
#pragma unroll
    for (int ky = 0; ky < 5; ++ky) tc::acc_fence<16>(acc[ky]);
    tc::mbar_arrive(&s.empty[st]);
  }
#pragma unroll
  for (int ky = 0; ky < 5; ++ky) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int row = h * 64 + tc::acc_row(t, i), kx = row >> 4, ci = row & 15, co = tc::acc_col(t, i);   // row = kx*16 + ci
      if (co >= 20) continue;
      if (kx < 5 && ci < 10) atomicAdd(grads + W2 + co * 250 + ci * 25 + ky * 5 + kx, acc[ky][i]);
      else if (ky == 0 && kx == 0 && ci == 10) atomicAdd(grads + B2 + co, acc[ky][i]);
    }
  }
}

// =====================================================================================================================
// conv2 data gradient on wgmma + col2im + relu/pool backward of conv1:
//   dA[(b, pos), (tap, ci)] = sum_co dC[b, co, pos] * W2[co, ci, tap]         M = 128 (2 samples), N = 400, K = 32
//   dP1[b, ci, y, x] = sum_{ky,kx} dA[(b, (y-ky, x-kx)), (ky*5+kx, ci)]       gathered from a bf16 staging tile
//   G1 = dP1 masked by relu(conv1-pool) > 0                                    fp32 [B,10,144]
// =====================================================================================================================
constexpr int DG_ROW = 816;                            // staging row stride in bytes (conflict-free for 16-byte accesses)
constexpr int DG_NC = 80;                              // N = 400 as 5 instructions of N = 80 (40 accumulator registers)
struct __align__(1024) DgSmem {
  uint8_t w[W2R_N * 128];                              // W2R [400 rows (tap, ci)][64 k (co)] K-major
  uint8_t a[2][8192];                                  // dC of 2 samples: [b][32 co][64 pos] = MN-major A (K = co)
  uint8_t stg[128 * DG_ROW];
  uint64_t full[2], empty[2], wfull;
};

__global__ void __launch_bounds__(BT_THREADS, 1)
bt_conv2_dgrad(const __grid_constant__ CUtensorMap map_dc, const __grid_constant__ CUtensorMap map_w2r, int B,
               const unsigned char* __restrict__ A1, float* __restrict__ G1) {
  extern __shared__ uint8_t smem_raw[];
  DgSmem& s = *reinterpret_cast<DgSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int tiles = (B + 1) / 2;
  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&map_dc); tc::prefetch_tmap(&map_w2r);
    for (int i = 0; i < 2; ++i) { tc::mbar_init(&s.full[i], 1); tc::mbar_init(&s.empty[i], 256); }
    tc::mbar_init(&s.wfull, 1);
    tc::mbar_fence_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (t == 0) {
      tc::mbar_expect_tx(&s.wfull, W2R_N * 128);
      tc::tma_load_2d(s.w, &map_w2r, &s.wfull, 0, 0);
      tc::tma_load_2d(s.w + 200 * 128, &map_w2r, &s.wfull, 0, 200);
      uint32_t it = 0;
      for (int tt = blockIdx.x; tt < tiles; tt += gridDim.x, ++it) {
        const int st = it & 1;
        tc::mbar_wait(&s.empty[st], ((it >> 1) & 1) ^ 1);
        tc::mbar_expect_tx(&s.full[st], 8192);
        tc::tma_load_2d(s.a[st], &map_dc, &s.full[st], 0, 64 * tt);
      }
    }
    return;
  }
  // warpgroup h: sample h of the tile = accumulator rows (positions) 0..63, staged as bf16 rows 64h..64h+63
  const int h = wg - 1, e = threadIdx.x - 128;            // e: 0..255
  tc::mbar_wait(&s.wfull, 0);
  uint32_t it = 0;
  for (int tt = blockIdx.x; tt < tiles; tt += gridDim.x, ++it) {
    const int b0 = 2 * tt, st = it & 1;
    tc::mbar_wait(&s.full[st], (it >> 1) & 1);
    const uint32_t a0 = tc::smem_u32(s.a[st]) + h * 4096, w0 = tc::smem_u32(s.w);
#pragma unroll 1
    for (int c0 = 0; c0 < W2R_N; c0 += DG_NC) {
      float d[DG_NC / 2];
#pragma unroll
      for (int i = 0; i < DG_NC / 2; ++i) d[i] = 0.f;
      tc::wg_fence();
#pragma unroll
      for (int ks = 0; ks < 2; ++ks)
        tc::mma<DG_NC>(d, tc::smem_desc(a0 + ks * 2048, /*LBO: next sample*/ 4096, 1024, tc::kSw128),
                       tc::smem_desc(w0 + c0 * 128 + ks * 32, 16, 1024, tc::kSw128), ks, /*A MN-major*/ 1u);
      tc::wg_commit();
      tc::wg_wait_all();
      tc::acc_fence<DG_NC / 2>(d);
#pragma unroll
      for (int i = 0; i < DG_NC / 2; i += 2) {
        const int row = h * 64 + tc::acc_row(t, i), col = c0 + tc::acc_col(t, i);
        *reinterpret_cast<uint32_t*>(s.stg + row * DG_ROW + col * 2) = b2::pack_bf16x2(d[i], d[i + 1]);
      }
    }
    tc::mbar_arrive(&s.empty[st]);
    tc::named_bar_sync(1, 256);
    // col2im gather: item = (sample in tile, y, x) of the 12 x 12 conv1 map
    for (int item = e; item < 288; item += 256) {
      const int sb = item / 144, p = item % 144, y = p / 12, x = p % 12;
      float acc[10];
#pragma unroll
      for (int c = 0; c < 10; ++c) acc[c] = 0.f;
#pragma unroll
      for (int ky = 0; ky < 5; ++ky) {
        const int oy = y - ky;
        if ((unsigned)oy < 8u) {
#pragma unroll
          for (int kx = 0; kx < 5; ++kx) {
            const int ox = x - kx;
            if ((unsigned)ox < 8u) {
              const uint8_t* src = s.stg + (sb * 64 + oy * 8 + ox) * DG_ROW + (ky * 5 + kx) * 32;
              const uint4 u0 = *reinterpret_cast<const uint4*>(src);
              const uint32_t u1 = *reinterpret_cast<const uint32_t*>(src + 16);
              acc[0] += b2::bf16lo(u0.x); acc[1] += b2::bf16hi(u0.x); acc[2] += b2::bf16lo(u0.y); acc[3] += b2::bf16hi(u0.y);
              acc[4] += b2::bf16lo(u0.z); acc[5] += b2::bf16hi(u0.z); acc[6] += b2::bf16lo(u0.w); acc[7] += b2::bf16hi(u0.w);
              acc[8] += b2::bf16lo(u1); acc[9] += b2::bf16hi(u1);
            }
          }
        }
      }
      if (b0 + sb < B) {
#pragma unroll
        for (int c = 0; c < 10; ++c) {
          const unsigned char code = __ldg(A1 + (size_t)(b0 + sb) * 1440 + c * 144 + p);
          G1[(size_t)(b0 + sb) * 1440 + c * 144 + p] = (code & 4) ? 0.f : acc[c];
        }
      }
    }
    tc::named_bar_sync(1, 256);                                  // staging tile free for the next tile
  }
}

// =====================================================================================================================
// conv1 weight/bias gradient (sparse: the gradient of a pooled cell goes to its argmax position).
// Lane = (cell in a group of 3, channel): the 30 active lanes of a warp read 5x5 windows that start within a few pixels of
// each other, so the 25 shared-memory loads per item are (nearly) conflict-free -- the first version (lane = cell, warp =
// channel) spread a warp's windows over three image rows and ran 4-way bank-conflicted (89 us at B = 4096).  Each lane keeps
// the 25 taps + bias of ITS channel in registers over all samples of the CTA; one reduction at the end.
// =====================================================================================================================
constexpr int C1W_WARPS = 8;
__global__ void __launch_bounds__(C1W_WARPS * 32) bt_conv1_wgrad(const void* __restrict__ x, int x_u8, float mean, float inv_std,
                                                                  const float* __restrict__ G1, const unsigned char* __restrict__ A1,
                                                                  int B, float* __restrict__ grads) {
  constexpr int NT = C1W_WARPS * 32;
  __shared__ __align__(16) float xs[28 * 28 + 4];
  __shared__ __align__(16) float gs[144 * 11];             // [cell][channel], row stride 11: conflict-free for (3 cells x 10 ch)
  __shared__ unsigned char as[144 * 11];
  __shared__ float red[C1W_WARPS][10][26];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cl = lane / 10, c = lane - cl * 10;            // lanes 30, 31 idle
  float acc[25], bsum = 0.f;
#pragma unroll
  for (int k = 0; k < 25; ++k) acc[k] = 0.f;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    if (x_u8) {
      if (tid < 49) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const unsigned char*>(x) + (size_t)b * 784) + tid);
        const unsigned int wv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 16; ++e) xs[tid * 16 + e] = ((float)((wv[e >> 2] >> ((e & 3) * 8)) & 0xffu) * (1.f / 255.f) - mean) * inv_std;
      }
    } else {
      if (tid < 196) reinterpret_cast<float4*>(xs)[tid] = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(x) + (size_t)b * 784) + tid);
    }
    for (int i = tid; i < 1440; i += NT) {                 // coalesced read of [c][cell], transposed store
      const int ch = i / 144, cell = i - ch * 144;
      gs[cell * 11 + ch] = __ldg(G1 + (size_t)b * 1440 + i);
      as[cell * 11 + ch] = __ldg(A1 + (size_t)b * 1440 + i);
    }
    __syncthreads();
    if (lane < 30) {
      for (int cg = warp; cg < 48; cg += C1W_WARPS) {      // 48 groups of 3 consecutive cells
        const int cell = cg * 3 + cl;
        const float g = gs[cell * 11 + c];
        if (g != 0.f) {
          const int arg = as[cell * 11 + c] & 3;
          const float* src = &xs[(2 * (cell / 12) + (arg >> 1)) * 28 + 2 * (cell % 12) + (arg & 1)];
          bsum += g;
#pragma unroll
          for (int ky = 0; ky < 5; ++ky)
#pragma unroll
            for (int kx = 0; kx < 5; ++kx) acc[ky * 5 + kx] = fmaf(g, src[ky * 28 + kx], acc[ky * 5 + kx]);
        }
      }
    }
  }
  // lanes c, c + 10, c + 20 hold the same channel: fold them, then fold the warps, then one atomic per output per CTA
#pragma unroll
  for (int k = 0; k < 26; ++k) {
    float v = k < 25 ? acc[k < 25 ? k : 0] : bsum;
    const float v1 = __shfl_down_sync(0xffffffffu, v, 10), v2 = __shfl_down_sync(0xffffffffu, v, 20);
    if (lane < 10) red[warp][lane][k] = v + v1 + v2;
  }
  __syncthreads();
  for (int i = tid; i < 260; i += NT) {
    const int ch = i / 26, k = i - ch * 26;
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < C1W_WARPS; ++w) v += red[w][ch][k];
    atomicAdd(grads + (k < 25 ? W1 + ch * 25 + k : B1 + ch), v);
  }
}

// =====================================================================================================================
// fc1 / fc2 weight and bias gradients: register-tiled outer products over a chunk of samples per CTA.
//   threads 0..399   : dW3[5 j x 8 i] tiles (50 x 320)
//   threads 400..511 : flat list [dW4 (500) | db3 (50) | db4 (10)], 5 entries each
// =====================================================================================================================
constexpr int FW_TS = 16;     // samples per shared-memory tile
__global__ void __launch_bounds__(512) bt_fc_wgrad(const __nv_bfloat16* __restrict__ P2, const __nv_bfloat16* __restrict__ H,
                                                   const __nv_bfloat16* __restrict__ DH, const float* __restrict__ DLOG,
                                                   int B, int samples_per_cta, float* __restrict__ grads) {
  __shared__ __align__(16) float p2s[FW_TS][320];
  __shared__ __align__(16) float dhs[FW_TS][52];
  __shared__ __align__(16) float hs[FW_TS][52];
  __shared__ __align__(16) float dls[FW_TS][12];
  const int tid = threadIdx.x;
  const int jg = tid / 40, ig = tid % 40;
  float acc[40];
#pragma unroll
  for (int i = 0; i < 40; ++i) acc[i] = 0.f;
  const int u = tid - 400;
  const int s_begin = blockIdx.x * samples_per_cta, s_end = min(B, s_begin + samples_per_cta);
  for (int s0 = s_begin; s0 < s_end; s0 += FW_TS) {
    const int ns = min(FW_TS, s_end - s0);
    __syncthreads();
    for (int i = tid; i < FW_TS * 40; i += 512) {                  // P2 rows: 40 x uint4 (8 bf16)
      const int sl = i / 40, q = i % 40;
      float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (sl < ns) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(P2 + (size_t)(s0 + sl) * 320) + q);
        f[0] = b2::bf16lo(v.x); f[1] = b2::bf16hi(v.x); f[2] = b2::bf16lo(v.y); f[3] = b2::bf16hi(v.y);
        f[4] = b2::bf16lo(v.z); f[5] = b2::bf16hi(v.z); f[6] = b2::bf16lo(v.w); f[7] = b2::bf16hi(v.w);
      }
      reinterpret_cast<float4*>(&p2s[sl][q * 8])[0] = make_float4(f[0], f[1], f[2], f[3]);
      reinterpret_cast<float4*>(&p2s[sl][q * 8])[1] = make_float4(f[4], f[5], f[6], f[7]);
    }
    for (int i = tid; i < FW_TS * 52; i += 512) {
      const int sl = i / 52, j = i % 52;
      float dv = 0.f, hv = 0.f;
      if (sl < ns) {
        dv = __bfloat162float(DH[(size_t)(s0 + sl) * 64 + j]);
        hv = __bfloat162float(H[(size_t)(s0 + sl) * 64 + j]);
      }
      dhs[sl][j] = dv; hs[sl][j] = hv;
    }
    for (int i = tid; i < FW_TS * 12; i += 512) {
      const int sl = i / 12, k = i % 12;
      dls[sl][k] = sl < ns ? DLOG[(size_t)(s0 + sl) * 16 + k] : 0.f;
    }
    __syncthreads();
    if (tid < 400) {
#pragma unroll 4
      for (int sl = 0; sl < FW_TS; ++sl) {
        const float4 pa = *reinterpret_cast<const float4*>(&p2s[sl][ig * 8]), pb = *reinterpret_cast<const float4*>(&p2s[sl][ig * 8 + 4]);
        const float pv[8] = {pa.x, pa.y, pa.z, pa.w, pb.x, pb.y, pb.z, pb.w};
#pragma unroll
        for (int jj = 0; jj < 5; ++jj) {
          const float d = dhs[sl][jg * 5 + jj];
#pragma unroll
          for (int ii = 0; ii < 8; ++ii) acc[jj * 8 + ii] = fmaf(d, pv[ii], acc[jj * 8 + ii]);
        }
      }
    } else {
#pragma unroll
      for (int n = 0; n < 5; ++n) {
        const int idx = u * 5 + n;
        float a = acc[n];
        if (idx < 500) {
          const int k = idx / 50, j = idx % 50;
          for (int sl = 0; sl < FW_TS; ++sl) a = fmaf(dls[sl][k], hs[sl][j], a);
        } else if (idx < 550) {
          for (int sl = 0; sl < FW_TS; ++sl) a += dhs[sl][idx - 500];
        } else if (idx < 560) {
          for (int sl = 0; sl < FW_TS; ++sl) a += dls[sl][idx - 550];
        }
        acc[n] = a;
      }
    }
  }
  if (tid < 400) {
#pragma unroll
    for (int jj = 0; jj < 5; ++jj) {                    // W3 + j*320 + ig*8 is 16-byte aligned (W3 = 5284 = 4 * 1321)
      float* dst = grads + W3 + (jg * 5 + jj) * 320 + ig * 8;
      cn::red_add_v4(dst, acc[jj * 8], acc[jj * 8 + 1], acc[jj * 8 + 2], acc[jj * 8 + 3]);
      cn::red_add_v4(dst + 4, acc[jj * 8 + 4], acc[jj * 8 + 5], acc[jj * 8 + 6], acc[jj * 8 + 7]);
    }
  } else {
#pragma unroll
    for (int n = 0; n < 5; ++n) {
      const int idx = u * 5 + n;
      if (idx < 500) atomicAdd(grads + W4 + idx, acc[n]);
      else if (idx < 550) atomicAdd(grads + B3 + idx - 500, acc[n]);
      else if (idx < 560) atomicAdd(grads + B4 + idx - 550, acc[n]);
    }
  }
}

// =====================================================================================================================
// bf16 operand copies of the weights in the layouts the GEMMs read (after every optimizer step).
//   W2K [32 co][448 k]   k = tap*16 + ci             conv2 forward B operand
//   W2R [400 n][64 k]    n = tap*16 + ci, k = co     conv2 data-gradient B operand
//   W3K [64 j][320 i]                                fc1 forward B operand       (rows >= 50 zero)
//   W3T [320 i][64 j]                                fc1 data-gradient B operand (cols >= 50 zero)
//   B3P [64] fp32                                    fc1 bias padded
// =====================================================================================================================
__global__ void __launch_bounds__(256) bt_pack_weights(const float* __restrict__ params, __nv_bfloat16* __restrict__ W2K,
                                                       __nv_bfloat16* __restrict__ W2R, __nv_bfloat16* __restrict__ W3K,
                                                       __nv_bfloat16* __restrict__ W3T, float* __restrict__ B3P) {
  b2::pdl_wait();
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < 32 * W2K_K) {
    const int co = i / W2K_K, k = i % W2K_K, tap = k >> 4, ci = k & 15;
    W2K[i] = __float2bfloat16((co < 20 && tap < 25 && ci < 10) ? params[W2 + co * 250 + ci * 25 + tap] : 0.f);
  }
  if (i < W2R_N * 64) {
    const int n = i >> 6, co = i & 63, tap = n >> 4, ci = n & 15;
    W2R[i] = __float2bfloat16((co < 20 && ci < 10) ? params[W2 + co * 250 + ci * 25 + tap] : 0.f);
  }
  if (i < 64 * 320) {
    const int j = i / 320, ii = i % 320;
    W3K[i] = __float2bfloat16(j < 50 ? params[W3 + j * 320 + ii] : 0.f);
    const int i2 = i >> 6, j2 = i & 63;
    W3T[i] = __float2bfloat16(j2 < 50 ? params[W3 + j2 * 320 + i2] : 0.f);
  }
  if (i < 64) B3P[i] = i < 50 ? params[B3 + i] : 0.f;
}

// ----------------------------------------------------------------------------------------------------- host side
std::string g_err;
using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeFn get_encode() {
  static EncodeFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess) {
      cudaGetLastError();
      p = nullptr;
    }
    return reinterpret_cast<EncodeFn>(p);
  }();
  return fn;
}
bool encode(CUtensorMap* map, const void* ptr, int rank, const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box,
            CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeFn enc = get_encode();
  if (!enc) { g_err = "cuTensorMapEncodeTiled not available (no CUDA driver?)"; return false; }
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { g_err = "cuTensorMapEncodeTiled failed: " + std::to_string((int)r); return false; }
  return true;
}
// [y][b][x][c] image of two samples for the conv2-forward window descriptors: tensor dims ordered (c, x, b, y)
bool map_p1_ybxc(CUtensorMap* m, const void* p1, int B) {
  cuuint64_t dims[4] = {16, 12, (cuuint64_t)B, 12};
  cuuint64_t strides[3] = {32, 12 * 12 * 32, 12 * 32};
  cuuint32_t box[4] = {16, 12, 2, 12};
  return encode(m, p1, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_32B);
}
// whole [y][x][c] image of one sample (conv2 weight gradient)
bool map_p1_image(CUtensorMap* m, const void* p1, int B) {
  cuuint64_t dims[4] = {16, 12, 12, (cuuint64_t)B};
  cuuint64_t strides[3] = {32, 12 * 32, 12 * 12 * 32};
  cuuint32_t box[4] = {16, 12, 12, 1};
  return encode(m, p1, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_32B);
}
bool map_p1(CUtensorMap* m, const void* p1, int B, int box_b) {
  // NHWC [B][12 y][12 x][16 c]: the innermost box start (channel 0) is always 16-byte aligned; kx / ky shift dims 1 / 2
  cuuint64_t dims[4] = {16, 12, 12, (cuuint64_t)B};
  cuuint64_t strides[3] = {32, 12 * 32, 12 * 12 * 32};
  cuuint32_t box[4] = {16, 8, 8, (cuuint32_t)box_b};
  return encode(m, p1, 4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_32B);
}
bool map_rows(CUtensorMap* m, const void* ptr, long long rows, int cols, int box_rows) {   // [rows][cols] bf16, box {64, box_rows}
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  return encode(m, ptr, 2, dims, strides, box);
}
int sm_count() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}

}  // namespace bt

extern "C" {

int b2_gemm_bf16_launch(const void* a, const void* b, void* c, const float* bias, int M, int N, int K, int relu, int out_bf16,
                        cudaStream_t stream);
const char* b2_gemm_last_error();

const char* b2_bt_last_error() { return bt::g_err.c_str(); }

struct BtBuffers {
  __nv_bfloat16 *P1, *P2, *H, *DH, *dP2, *DC, *W2K, *W2R, *W3K, *W3T;
  unsigned char *A1, *A2;
  float *Hrelu, *DLOG, *G1, *B3P;
};

int b2_bt_pack_weights(const float* params, const BtBuffers* bf, cudaStream_t stream) {
  const int n = bt::W2R_N * 64;   // largest of the four
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)((n + 255) / 256));
  cfg.blockDim = dim3(256);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return (int)cudaLaunchKernelEx(&cfg, bt::bt_pack_weights, params, bf->W2K, bf->W2R, bf->W3K, bf->W3T, bf->B3P);
}

// One forward (+ backward) pass over a batch.  `grads` must be zero on entry (the optimizer kernel re-zeroes it).
// stage_mask selects kernels (tests): bit0 conv1_fwd, bit1 conv2_fwd, bit2 fc1+head, bit3 fc1 dgrad+route, bit4 conv2 wgrad,
// bit5 conv2 dgrad, bit6 conv1 wgrad, bit7 fc wgrad.
int b2_bt_step_launch(const float* params, float* grads, const void* x, int x_u8, const long long* target, const BtBuffers* bf,
                      float* loss_acc, float* out_logp, const unsigned long long* step, unsigned long long seed,
                      long long sample_base, int B, int training, int backward, float inv_bsz, float p_drop, int stage_mask,
                      cudaStream_t stream) {
  using namespace bt;
  if (B < 1) { g_err = "empty batch"; return -1; }
  static bool configured = false;
  const size_t sm_c2f = sizeof(C2fSmem) + 1024, sm_wg = sizeof(WgSmem) + 1024, sm_dg = sizeof(DgSmem) + 1024;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(bt_conv2_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_c2f);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(bt_conv2_wgrad, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_wg);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(bt_conv2_dgrad, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm_dg);
    if (e != cudaSuccess) { g_err = std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e); return -2; }
    configured = true;
  }
  Common cm;
  cm.seed = seed; cm.step = step; cm.sample_base = sample_base; cm.B = B; cm.training = training; cm.p_drop = p_drop;
  const float mean = 0.1307f, inv_std = 1.f / 0.3081f;
  const int sms = sm_count();
  CUtensorMap m_p1_2, m_p1_1, m_w2k, m_dc64, m_dc32, m_w2r;
  if (!map_p1_ybxc(&m_p1_2, bf->P1, B) || !map_p1_image(&m_p1_1, bf->P1, B) || !map_rows(&m_w2k, bf->W2K, 32, W2K_K, 32) ||
      !map_rows(&m_dc64, bf->DC, (long long)B * 32, 64, 64) || !map_rows(&m_dc32, bf->DC, (long long)B * 32, 64, 32) ||
      !map_rows(&m_w2r, bf->W2R, W2R_N, 64, 200))
    return -3;
  cudaError_t e = cudaSuccess;
  auto ck = [&](const char* what) {
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) { g_err = std::string(what) + ": " + cudaGetErrorString(e); return false; }
    return true;
  };
  if (stage_mask & 1) {
    const int pairs = (B + 1) / 2;
    bt_conv1_fwd<<<pairs < sms * 5 ? pairs : sms * 5, 288, 0, stream>>>(params, x, x_u8, mean, inv_std, B, bf->P1, bf->A1);
    if (!ck("conv1_fwd")) return -4;
  }
  if (stage_mask & 2) {
    const int tiles = (B + 1) / 2;
    bt_conv2_fwd<<<tiles < sms ? tiles : sms, BT_THREADS, sm_c2f, stream>>>(m_p1_2, m_w2k, params, cm, bf->P2, bf->A2);
    if (!ck("conv2_fwd")) return -4;
  }
  if (stage_mask & 4) {
    if (b2_gemm_bf16_launch(bf->P2, bf->W3K, bf->Hrelu, bf->B3P, B, 64, 320, 1, 0, stream) != 0) { g_err = std::string("fc1 gemm: ") + b2_gemm_last_error(); return -5; }
    bt_head<<<(B + 127) / 128, 128, 0, stream>>>(params, bf->Hrelu, target, cm, backward, inv_bsz, bf->H, bf->DH, bf->DLOG, loss_acc, out_logp);
    if (!ck("head")) return -4;
  }
  if (!backward) return 0;
  if (stage_mask & 8) {
    if (b2_gemm_bf16_launch(bf->DH, bf->W3T, bf->dP2, nullptr, B, 320, 64, 0, 1, stream) != 0) { g_err = std::string("fc1 dgrad gemm: ") + b2_gemm_last_error(); return -5; }
    bt_route<<<(B * 20 + 255) / 256, 256, 0, stream>>>(bf->dP2, bf->A2, B, training ? 1.f / (1.f - p_drop) : 1.f, bf->DC);
    if (!ck("route")) return -4;
  }
  // The four gradient kernels are independent after `route`.  Two branches (a side stream forked/joined with events; under
  // graph capture they become parallel graph branches):  main: conv2_dgrad -> conv1_wgrad    side: fc_wgrad -> conv2_wgrad
  // The SIMT kernels (small shared memory) co-reside with the tensor-core kernels (one CTA of up to ~175 KB per SM).
  static cudaStream_t side = nullptr;
  static cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  const bool overlap = (stage_mask & 255) == 255;
  if (overlap && side == nullptr) {
    cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking);
    cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming);
  }
  cudaStream_t s2 = overlap ? side : stream;
  if (overlap) { cudaEventRecord(ev_fork, stream); cudaStreamWaitEvent(side, ev_fork, 0); }
  if (stage_mask & 128) {
    const int per = B >= sms * 32 ? (B + sms - 1) / sms : 32;        // ~one CTA per SM; >= 32 samples amortise the final atomics
    const int ctas = (B + per - 1) / per;
    bt_fc_wgrad<<<ctas, 512, 0, s2>>>(bf->P2, bf->H, bf->DH, bf->DLOG, B, per, grads);
    if (!ck("fc_wgrad")) return -4;
  }
  if (stage_mask & 16) {
    bt_conv2_wgrad<<<B < sms ? B : sms, BT_THREADS, sm_wg, s2>>>(m_p1_1, m_dc32, B, grads);
    if (!ck("conv2_wgrad")) return -4;
  }
  if (stage_mask & 32) {
    const int tiles = (B + 1) / 2;
    bt_conv2_dgrad<<<tiles < sms ? tiles : sms, BT_THREADS, sm_dg, stream>>>(m_dc64, m_w2r, B, bf->A1, bf->G1);
    if (!ck("conv2_dgrad")) return -4;
  }
  if (stage_mask & 64) {
    bt_conv1_wgrad<<<B < sms * 4 ? B : sms * 4, C1W_WARPS * 32, 0, stream>>>(x, x_u8, mean, inv_std, bf->G1, bf->A1, B, grads);
    if (!ck("conv1_wgrad")) return -4;
  }
  if (overlap) { cudaEventRecord(ev_join, side); cudaStreamWaitEvent(stream, ev_join, 0); }
  return 0;
}

}  // extern "C"
