// Fused MNIST-ConvNet training step, ONE THREAD-BLOCK CLUSTER PER SAMPLE (strong-scaling variant of convnet.cu).
//
// The reference keeps the global batch at 128 (`bsz = 128 // world_size`, train_dist.py:85), so with N GPUs each GPU
// only has 128/N samples: one CTA per sample (convnet.cu) leaves most of the SMs idle and the step time is the
// latency of a single sample (~30 us) no matter how many GPUs are used.  Here a sample is carried by a cluster of C CTAs
// (C = 2, 4, 8 on as many SMs): every phase of the forward/backward pass is split C ways, the small activations every CTA
// needs next (pooled conv outputs, fc1 activations, their gradients) are broadcast into all peers' shared memory with
// distributed-shared-memory stores, and a cluster barrier (barrier.cluster arrive.release / wait.acquire) separates the
// phases (4 per sample; fc1/fc2 and their small backward pieces are recomputed by every CTA instead of exchanged).  Weights are staged by every CTA (parallel L2 reads); each CTA flushes only the gradient slices it owns, so the
// number of global `red.add` operations per sample stays 21,848 but is issued from C SMs at once.
#include <cooperative_groups.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "convnet_args.cuh"

namespace cg = cooperative_groups;

namespace cnc {

using namespace cn;
constexpr int T = 512;

template <int C>
struct Cfg {
  static constexpr int P1_PER = 1440 / C;            // conv1 pooled outputs per CTA
  static constexpr int TILES = 80 / C;               // conv2 (cell, 4-channel group) tiles per CTA
  static constexpr int FC1_PER = (50 + C - 1) / C;   // fc1 outputs per CTA
  static constexpr int P2_PER = 320 / C;             // fc1-input gradient entries per CTA
  static constexpr int W4_PER = (500 + C - 1) / C;
  static constexpr int W2_PER = 5000 / C;            // conv2.weight gradient entries per CTA
  static constexpr int UNITS = 72 / C;               // dgrad (2x2 tile, 5-channel half) units per CTA
  static constexpr int KS_D = C == 2 ? 10 : 20;      // dgrad split over output channels inside the CTA
  static constexpr int W1_PER = (250 + C - 1) / C;   // conv1.weight gradient entries per CTA
};

struct __align__(16) Smem {
  float w1[252];
  float b1[12];
  float b2[20];
  float w4[500];
  float b4[12];
  float w2f[250 * 20];      // [ci][ky][kx][co]
  float w2b[500 * 16];      // [co][ky][kx][half][8]
  float x[784];
  float p1[P1_SIZE];        // padded strides, see convnet_args.cuh
  float p2[320];
  float g2[320];
  float2 g1[1440];
  float h[52];
  float hm[52];
  float dh[52];
  float dlog[12];
  float m2[20];
  float rnd[72];
  float part[7200];         // conv2 split-K partials / dgrad split-K partials
  float dc2pad[DC_SIZE];   
  float g[NPAR];
  unsigned char a1[1440];
  unsigned char a2[320];
  float loss_local;
  int correct_local;
};

template <int C, typename V>
__device__ __forceinline__ void bcast(cg::cluster_group& cl, V* local, V v) {
#pragma unroll
  for (int r = 0; r < C; ++r) *cl.map_shared_rank(local, r) = v;
}

template <int C>
__global__ void __launch_bounds__(T, 1) convnet_cluster_kernel(Args a) {
  using K = Cfg<C>;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  cg::cluster_group cl = cg::this_cluster();
  const int tid = threadIdx.x;
  const int cr = (int)cl.block_rank();
  const int cluster_id = blockIdx.x / C, n_clusters = gridDim.x / C;
  const float* __restrict__ P = a.params;

  // ---------------------------------------------------------------- P0: stage weights (every CTA), zero accumulators
  b2::pdl_launch_dependents();
  {
    float4* g4 = reinterpret_cast<float4*>(s.g);
    for (int i = tid; i < NPAR / 4; i += T) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  b2::pdl_wait();
  {
    const bool fast = (a.aux != nullptr);   // conv2.weight already in both smem layouts (written by sgd.cu)
    float4 fa[3], fb[4];            // pre-arranged conv2.weight: every load is in flight before the first store
    if (fast) {
      const float4* __restrict__ af = reinterpret_cast<const float4*>(a.aux + AUX_W2F);
      const float4* __restrict__ ab = reinterpret_cast<const float4*>(a.aux + AUX_W2B);
#pragma unroll
      for (int k = 0; k < 3; ++k) fa[k] = (tid + k * T < 1250) ? __ldg(af + tid + k * T) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int k = 0; k < 4; ++k) fb[k] = (tid + k * T < 2000) ? __ldg(ab + tid + k * T) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const float4* __restrict__ P4w2 = reinterpret_cast<const float4*>(P + W2);
    float4 v[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int i4 = tid + k * T;
      v[k] = (!fast && i4 < 1250) ? __ldg(P4w2 + i4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const float w1v = tid < 250 ? __ldg(P + W1 + tid) : 0.f;
    const float w4v = tid < 500 ? __ldg(P + W4 + tid) : 0.f;
    const float bv = tid < 10 ? __ldg(P + B1 + tid) : (tid < 20 ? __ldg(P + B4 + tid - 10) : (tid < 40 ? __ldg(P + B2 + tid - 20) : 0.f));
    if (tid < 250) s.w1[tid] = w1v;
    if (tid < 500) s.w4[tid] = w4v;
    if (tid < 10) s.b1[tid] = bv; else if (tid < 20) s.b4[tid - 10] = bv; else if (tid < 40) s.b2[tid - 20] = bv;
    if (fast) {
      float4* df = reinterpret_cast<float4*>(s.w2f);
      float4* db = reinterpret_cast<float4*>(s.w2b);
#pragma unroll
      for (int k = 0; k < 3; ++k) if (tid + k * T < 1250) df[tid + k * T] = fa[k];
#pragma unroll
      for (int k = 0; k < 4; ++k) if (tid + k * T < 2000) db[tid + k * T] = fb[k];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int i4 = tid + k * T;
      if (!fast && i4 < 1250) {
        const float w[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int i = i4 * 4 + e;
          const int co = i / 250, r = i % 250, ci = r / 25, kk = r % 25;
          s.w2f[(ci * 25 + kk) * 20 + co] = w[e];
          s.w2b[((co * 25 + kk) * 2 + ci / 5) * 8 + ci % 5] = w[e];
        }
      }
    }
    }
  if (tid == 0) { s.loss_local = 0.f; s.correct_local = 0; }
  const unsigned long long step = a.step ? *a.step : 0ull;
  const float keep_scale = 1.f / (1.f - a.p_drop);
  cl.sync();                                       // every CTA of the cluster is running (DSMEM stores may begin)

  for (int b = cluster_id; b < a.B; b += n_clusters) {
    // -------------------------------------------------------------- S0: input, RNG (every CTA), clear scratch
    if (a.x_u8) {
      const uint4* xs = reinterpret_cast<const uint4*>(reinterpret_cast<const unsigned char*>(a.x) + (size_t)b * 784);
      if (tid < 49) {
        const uint4 q = __ldcg(xs + tid);
        const unsigned int wv[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int e = 0; e < 16; ++e)
          s.x[tid * 16 + e] = ((float)((wv[e >> 2] >> ((e & 3) * 8)) & 0xffu) * (1.f / 255.f) - a.mean) * a.inv_std;
      }
    } else {
      const float4* xs = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(a.x) + (size_t)b * 784);
      if (tid < 196) reinterpret_cast<float4*>(s.x)[tid] = __ldcg(xs + tid);
    }
    if (tid >= 256 && tid < 274) {
      const int q = tid - 256;
      uint4 r = b2::Philox::gen(a.seed, (unsigned long long)(a.sample_base + b), step * 32ull + q);
      const float k = 2.3283064365386963e-10f;
      s.rnd[q * 4 + 0] = r.x * k; s.rnd[q * 4 + 1] = r.y * k;
      s.rnd[q * 4 + 2] = r.z * k; s.rnd[q * 4 + 3] = r.w * k;
    }
    for (int i = tid; i < DC_SIZE / 4; i += T) reinterpret_cast<float4*>(s.dc2pad)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    if (tid < 20) s.m2[tid] = a.training ? (s.rnd[tid] >= a.p_drop ? keep_scale : 0.f) : 1.f;

    // -------------------------------------------------------------- S1: conv1 -> pool -> relu  (1440 / C outputs, broadcast)
    for (int l = tid; l < K::P1_PER; l += T) {
      const int o = cr * K::P1_PER + l;
      const int c = o / 144, r = o % 144, py = r / 12, px = r % 12;
      float patch[6][6];
#pragma unroll
      for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {              // 8-byte aligned pairs: 18 LDS.64 instead of 36 LDS.32
          const float2 q = *reinterpret_cast<const float2*>(&s.x[(2 * py + i) * 28 + 2 * px + 2 * j]);
          patch[i][2 * j] = q.x; patch[i][2 * j + 1] = q.y;
        }
      const float bias = s.b1[c];
      float a00 = bias, a01 = bias, a10 = bias, a11 = bias;
#pragma unroll
      for (int ky = 0; ky < 5; ++ky)
#pragma unroll
        for (int kx = 0; kx < 5; ++kx) {
          const float w = s.w1[c * 25 + ky * 5 + kx];
          a00 = fmaf(w, patch[ky][kx], a00);
          a01 = fmaf(w, patch[ky][kx + 1], a01);
          a10 = fmaf(w, patch[ky + 1][kx], a10);
          a11 = fmaf(w, patch[ky + 1][kx + 1], a11);
        }
      float m = a00; int arg = 0;
      if (a01 > m) { m = a01; arg = 1; }
      if (a10 > m) { m = a10; arg = 2; }
      if (a11 > m) { m = a11; arg = 3; }
      bcast<C>(cl, &s.p1[p1_idx(c, py, px)], fmaxf(m, 0.f));
      bcast<C>(cl, &s.a1[o], (unsigned char)arg);
    }
    cl.sync();                                     // (1) p1 / a1 complete everywhere

    // -------------------------------------------------------------- S2: conv2, 80/C (cell, 4-channel) tiles x 10 input channels
    if (tid < K::TILES * 10) {
      const int tl = tid % K::TILES, ci = tid / K::TILES;
      const int tg = cr * K::TILES + tl, cell = tg & 15, cgp = tg >> 4;
      const int py = cell >> 2, px = cell & 3;
      float acc[4][4];
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[p][c] = 0.f;
      float patch[6][6];
      const float* src = &s.p1[p1_idx(ci, 2 * py, 2 * px)];
#pragma unroll
      for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j < 6; ++j) patch[i][j] = src[i * P1_ROW + j];
#pragma unroll
      for (int ky = 0; ky < 5; ++ky)
#pragma unroll
        for (int kx = 0; kx < 5; ++kx) {
          const float4 w = *reinterpret_cast<const float4*>(&s.w2f[((ci * 5 + ky) * 5 + kx) * 20 + cgp * 4]);
          const float i00 = patch[ky][kx], i01 = patch[ky][kx + 1], i10 = patch[ky + 1][kx], i11 = patch[ky + 1][kx + 1];
          acc[0][0] = fmaf(w.x, i00, acc[0][0]); acc[0][1] = fmaf(w.y, i00, acc[0][1]);
          acc[0][2] = fmaf(w.z, i00, acc[0][2]); acc[0][3] = fmaf(w.w, i00, acc[0][3]);
          acc[1][0] = fmaf(w.x, i01, acc[1][0]); acc[1][1] = fmaf(w.y, i01, acc[1][1]);
          acc[1][2] = fmaf(w.z, i01, acc[1][2]); acc[1][3] = fmaf(w.w, i01, acc[1][3]);
          acc[2][0] = fmaf(w.x, i10, acc[2][0]); acc[2][1] = fmaf(w.y, i10, acc[2][1]);
          acc[2][2] = fmaf(w.z, i10, acc[2][2]); acc[2][3] = fmaf(w.w, i10, acc[2][3]);
          acc[3][0] = fmaf(w.x, i11, acc[3][0]); acc[3][1] = fmaf(w.y, i11, acc[3][1]);
          acc[3][2] = fmaf(w.z, i11, acc[3][2]); acc[3][3] = fmaf(w.w, i11, acc[3][3]);
        }
      // part[ci][tile_local][channel c][4 window positions]
#pragma unroll
      for (int c = 0; c < 4; ++c)
        *reinterpret_cast<float4*>(&s.part[(ci * K::TILES + tl) * 16 + c * 4]) = make_float4(acc[0][c], acc[1][c], acc[2][c], acc[3][c]);
    }
    __syncthreads();
    if (tid < K::TILES * 4) {                      // +bias, dropout2d, pool, relu -> p2 entries of this CTA, broadcast
      const int tl = tid >> 2, c = tid & 3;
      const int tg = cr * K::TILES + tl, cell = tg & 15, co = (tg >> 4) * 4 + c;
      float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int ci = 0; ci < 10; ++ci) {
        const float4 t = *reinterpret_cast<const float4*>(&s.part[(ci * K::TILES + tl) * 16 + c * 4]);
        q.x += t.x; q.y += t.y; q.z += t.z; q.w += t.w;
      }
      const float bias = s.b2[co], sc = s.m2[co];
      const float v0 = (q.x + bias) * sc, v1 = (q.y + bias) * sc, v2 = (q.z + bias) * sc, v3 = (q.w + bias) * sc;
      float m = v0; int arg = 0;
      if (v1 > m) { m = v1; arg = 1; }
      if (v2 > m) { m = v2; arg = 2; }
      if (v3 > m) { m = v3; arg = 3; }
      const int o = co * 16 + cell;
      bcast<C>(cl, &s.p2[o], fmaxf(m, 0.f));
      bcast<C>(cl, &s.a2[o], (unsigned char)arg);
    }
    cl.sync();                                     // (2) p2 / a2 complete everywhere

    // -------------------------------------------------------------- S3: fc1 + relu + dropout (redundant in every CTA:
    //                                                                 16 k MACs cost less than a broadcast + cluster barrier)
    {
      const int j = tid >> 3, l8 = tid & 7;
      float sum = 0.f;
      if (j < 50) {
        const float4* wrow = reinterpret_cast<const float4*>(P + W3 + j * 320);
#pragma unroll
        for (int k = 0; k < 10; ++k) {
          const float4 w = __ldg(wrow + l8 + 8 * k);
          const float4 vv = *reinterpret_cast<const float4*>(&s.p2[(l8 + 8 * k) * 4]);
          sum = fmaf(w.x, vv.x, sum); sum = fmaf(w.y, vv.y, sum);
          sum = fmaf(w.z, vv.z, sum); sum = fmaf(w.w, vv.w, sum);
        }
      }
      sum += __shfl_xor_sync(0xffffffffu, sum, 4);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      if (j < 50 && l8 == 0) {
        const float pre = sum + __ldg(P + B3 + j);
        const float dm = a.training ? (s.rnd[20 + j] >= a.p_drop ? keep_scale : 0.f) : 1.f;
        s.h[j] = fmaxf(pre, 0.f) * dm;
        s.hm[j] = pre > 0.f ? dm : 0.f;
      }
    }
    __syncthreads();

    // -------------------------------------------------------------- S4: fc2 + log_softmax + nll (redundant in every CTA)
    if (tid < 32) {
      const long long y = __ldcg(a.target + b);
      float logit = -INFINITY;
      if (tid < 10) {
        float acc = s.b4[tid];
#pragma unroll 10
        for (int i = 0; i < 50; ++i) acc = fmaf(s.w4[tid * 50 + i], s.h[i], acc);
        logit = acc;
      }
      float mx = logit; int am = tid;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) {
        const float o = __shfl_xor_sync(0xffffffffu, mx, d);
        const int oi = __shfl_xor_sync(0xffffffffu, am, d);
        if (o > mx || (o == mx && oi < am)) { mx = o; am = oi; }
      }
      float e = tid < 10 ? __expf(logit - mx) : 0.f;
      float se = e;
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) se += __shfl_xor_sync(0xffffffffu, se, d);
      const float lse = mx + __logf(se);
      if (tid < 10) {
        const float logp = logit - lse;
        if (a.out_logp && cr == 0) a.out_logp[(size_t)b * 10 + tid] = logp;
        s.dlog[tid] = (e / se - (tid == (int)y ? 1.f : 0.f)) * a.inv_bsz;
        if (tid == (int)y && cr == 0) s.loss_local += -logp;
      }
      if (tid == 0 && am == (int)y && cr == 0) s.correct_local += 1;
    }
    if (a.mask_out && cr == 0) {
      if (tid < 20) a.mask_out[(size_t)b * 70 + tid] = s.m2[tid];
      else if (tid < 70) a.mask_out[(size_t)b * 70 + tid] = a.training ? (s.rnd[tid] >= a.p_drop ? keep_scale : 0.f) : 1.f;
    }
    __syncthreads();
    if (!a.backward) {                             // keep the cluster in lock-step before buffers are reused
      if (b + n_clusters < a.B) cl.sync();
      continue;
    }

    // -------------------------------------------------------------- S5: fc2 backward (weight slice of this CTA; dh everywhere)
    if (tid < K::W4_PER) {
      const int e = cr * K::W4_PER + tid;
      if (e < 500) s.g[W4 + e] += s.dlog[e / 50] * s.h[e % 50];
    }
    if (cr == 0 && tid >= 480 && tid < 490) s.g[B4 + tid - 480] += s.dlog[tid - 480];
    if (tid >= 64 && tid < 114) {
      const int i = tid - 64;
      float d = 0.f;
#pragma unroll
      for (int k = 0; k < 10; ++k) d = fmaf(s.w4[k * 50 + i], s.dlog[k], d);
      s.dh[i] = d * s.hm[i];
    }
    __syncthreads();

    // -------------------------------------------------------------- S6: fc1 backward (rows / input slices of this CTA)
    {
      float4* gw3 = reinterpret_cast<float4*>(&s.g[W3]);
      const float4* p24 = reinterpret_cast<const float4*>(s.p2);
      for (int l = tid; l < K::FC1_PER * 80; l += T) {
        const int jl = l / 80, i4 = l - jl * 80, j = cr * K::FC1_PER + jl;
        if (j < 50) {
          const float d = s.dh[j];
          const float4 pv = p24[i4];
          float4 gv = gw3[j * 80 + i4];
          gv.x = fmaf(d, pv.x, gv.x); gv.y = fmaf(d, pv.y, gv.y); gv.z = fmaf(d, pv.z, gv.z); gv.w = fmaf(d, pv.w, gv.w);
          gw3[j * 80 + i4] = gv;
        }
      }
      if (tid >= 448 && tid < 448 + K::FC1_PER) {
        const int j = cr * K::FC1_PER + tid - 448;
        if (j < 50) s.g[B3 + j] += s.dh[j];
      }
      // dp2 entries owned by this CTA: 4 lanes per entry over the 50 fc1 rows (warp-uniform trip count)
      for (int base = 0; base < K::P2_PER; base += T / 4) {
        const int ol = base + (tid >> 2), l4 = tid & 3, o = cr * K::P2_PER + ol;
        float d = 0.f;
        if (ol < K::P2_PER) {
          for (int jj = l4; jj < 50; jj += 4) d = fmaf(__ldg(P + W3 + jj * 320 + o), s.dh[jj], d);
        }
        d += __shfl_xor_sync(0xffffffffu, d, 2);
        d += __shfl_xor_sync(0xffffffffu, d, 1);
        if (ol < K::P2_PER && l4 == 0) {
          const int co = o >> 4;
          bcast<C>(cl, &s.g2[o], s.p2[o] > 0.f ? d * s.m2[co] : 0.f);
        }
      }
    }
    cl.sync();                                     // (4) g2 complete everywhere

    // -------------------------------------------------------------- S7: conv2 backward
    for (int o = tid; o < 320; o += T) {            // zero-padded conv2-output gradient (every CTA builds its own copy)
      const int co = o >> 4, cell = o & 15, arg = s.a2[o];
      const int y = 2 * (cell >> 2) + (arg >> 1), x = 2 * (cell & 3) + (arg & 1);
      s.dc2pad[co * DC_PLANE + (y + 4) * DC_ROW + (x + 4)] = s.g2[o];
    }
    // weight gradient: 5000 / C entries (co, ci, ky, kx), 16 pooled cells each
    for (int l = tid; l < K::W2_PER; l += T) {
      const int e = cr * K::W2_PER + l;
      const int co = e / 250, r = e - co * 250, ci = r / 25, k = r - ci * 25, ky = k / 5, kx = k - ky * 5;
      float acc = 0.f;
#pragma unroll 4
      for (int cell = 0; cell < 16; ++cell) {
        const float gv = s.g2[co * 16 + cell];
        const int arg = s.a2[co * 16 + cell];
        const int ay = 2 * (cell >> 2) + (arg >> 1), ax = 2 * (cell & 3) + (arg & 1);
        acc = fmaf(gv, s.p1[p1_idx(ci, ay + ky, ax + kx)], acc);
      }
      s.g[W2 + e] += acc;
    }
    if (cr == 0 && tid >= 480 && tid < 500) {
      const int co = tid - 480;
      float d = 0.f;
#pragma unroll
      for (int cell = 0; cell < 16; ++cell) d += s.g2[co * 16 + cell];
      s.g[B2 + co] += d;
    }
    __syncthreads();                               // dc2pad complete
    // data gradient: 72 / C (2x2 tile, 5-channel half) units x KS_D output-channel slices
    if (tid < K::UNITS * K::KS_D) {
      const int ul = tid % K::UNITS, ks = tid / K::UNITS;
      const int ug = cr * K::UNITS + ul, tile = ug % 36, half = ug / 36;
      const int y0 = 2 * (tile / 6), x0 = 2 * (tile % 6);
      constexpr int CO_PER = 20 / K::KS_D;
      float acc[4][5];
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int c = 0; c < 5; ++c) acc[p][c] = 0.f;
#pragma unroll 1
      for (int co = ks * CO_PER; co < (ks + 1) * CO_PER; ++co) {
        if (s.m2[co] == 0.f) continue;
        float patch[6][6];
        const float2* src = reinterpret_cast<const float2*>(&s.dc2pad[co * DC_PLANE + y0 * DC_ROW + x0]);   // even offsets
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
          for (int j = 0; j < 3; ++j) {
            const float2 q = src[i * (DC_ROW / 2) + j];
            patch[i][2 * j] = q.x; patch[i][2 * j + 1] = q.y;
          }
#pragma unroll
        for (int ky = 0; ky < 5; ++ky)
#pragma unroll
          for (int kx = 0; kx < 5; ++kx) {
            const float* wp = &s.w2b[((co * 25 + ky * 5 + kx) * 2 + half) * 8];
            const float4 w = *reinterpret_cast<const float4*>(wp);
            const float w4 = wp[4];
            const float d00 = patch[4 - ky][4 - kx], d01 = patch[4 - ky][5 - kx];
            const float d10 = patch[5 - ky][4 - kx], d11 = patch[5 - ky][5 - kx];
            acc[0][0] = fmaf(w.x, d00, acc[0][0]); acc[0][1] = fmaf(w.y, d00, acc[0][1]);
            acc[0][2] = fmaf(w.z, d00, acc[0][2]); acc[0][3] = fmaf(w.w, d00, acc[0][3]); acc[0][4] = fmaf(w4, d00, acc[0][4]);
            acc[1][0] = fmaf(w.x, d01, acc[1][0]); acc[1][1] = fmaf(w.y, d01, acc[1][1]);
            acc[1][2] = fmaf(w.z, d01, acc[1][2]); acc[1][3] = fmaf(w.w, d01, acc[1][3]); acc[1][4] = fmaf(w4, d01, acc[1][4]);
            acc[2][0] = fmaf(w.x, d10, acc[2][0]); acc[2][1] = fmaf(w.y, d10, acc[2][1]);
            acc[2][2] = fmaf(w.z, d10, acc[2][2]); acc[2][3] = fmaf(w.w, d10, acc[2][3]); acc[2][4] = fmaf(w4, d10, acc[2][4]);
            acc[3][0] = fmaf(w.x, d11, acc[3][0]); acc[3][1] = fmaf(w.y, d11, acc[3][1]);
            acc[3][2] = fmaf(w.z, d11, acc[3][2]); acc[3][3] = fmaf(w.w, d11, acc[3][3]); acc[3][4] = fmaf(w4, d11, acc[3][4]);
          }
      }
      float* dst = &s.part[(ks * K::UNITS + ul) * 20];      // [ks][unit_local][pos 4][c 5]
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int c = 0; c < 5; ++c) dst[p * 5 + c] = acc[p][c];
    }
    __syncthreads();
    for (int t = tid; t < K::UNITS * 20; t += T) {  // reduce the slices, route through relu'/pool of conv1, broadcast
      const int ul = t / 20, pc = t - ul * 20, p = pc / 5, c = pc - p * 5;
      float d = 0.f;
#pragma unroll
      for (int ks = 0; ks < K::KS_D; ++ks) d += s.part[(ks * K::UNITS + ul) * 20 + pc];
      const int ug = cr * K::UNITS + ul, tile = ug % 36, half = ug / 36;
      const int y = 2 * (tile / 6) + (p >> 1), x = 2 * (tile % 6) + (p & 1);
      const int o = (half * 5 + c) * 144 + y * 12 + x, arg = s.a1[o];
      const int off = (2 * y + (arg >> 1)) * 28 + 2 * x + (arg & 1);
      bcast<C>(cl, &s.g1[o], make_float2(s.p1[p1_of(o)] > 0.f ? d : 0.f, __int_as_float(off)));
    }
    cl.sync();                                     // (5) g1 complete everywhere

    // -------------------------------------------------------------- S8: conv1 weight/bias gradient (16 lanes per tap)
    for (int base = 0; base < K::W1_PER; base += T / 16) {
      const int ol = base + (tid >> 4), l16 = tid & 15, out = cr * K::W1_PER + ol;
      const bool act = ol < K::W1_PER && out < 250;
      float acc = 0.f, gsum = 0.f;
      int k = 1;
      if (act) {
        const int c = out / 25;
        k = out - c * 25;
        const int koff = (k / 5) * 28 + (k % 5);
        const float2* gp = &s.g1[c * 144 + l16 * 9];
#pragma unroll
        for (int cell = 0; cell < 9; ++cell) {
          const float2 q = gp[cell];
          gsum += q.x;
          acc = fmaf(q.x, s.x[__float_as_int(q.y) + koff], acc);
        }
      }
#pragma unroll
      for (int d = 8; d > 0; d >>= 1) {
        acc += __shfl_xor_sync(0xffffffffu, acc, d);
        gsum += __shfl_xor_sync(0xffffffffu, gsum, d);
      }
      if (act && l16 == 0) {
        s.g[W1 + out] += acc;
        if (k == 0) s.g[B1 + out / 25] += gsum;
      }
    }
    if (b + n_clusters < a.B) cl.sync();           // (6) nobody still reads buffers the next sample's broadcasts overwrite
  }

  // ------------------------------------------------------------------ flush: only the gradient slices this CTA owns
  __syncthreads();                                 // S8 of the last sample wrote s.g[W1..], s.g[B1..] from other warps (barrier (6) is
                                                   // skipped after the last sample; found by racecheck)
  if (a.backward && cluster_id < a.B) {
    float* gdst = a.grads + (size_t)(step & 1ull) * (size_t)a.grad_stride;
    if (a.det_partials != nullptr) {               // deterministic mode: whole private slot per CTA (zeros outside its slices)
      float4* slot = reinterpret_cast<float4*>(a.det_partials + (size_t)blockIdx.x * DET_STRIDE);
      for (int v = tid; v < NPAR / 4; v += T) slot[v] = *reinterpret_cast<const float4*>(&s.g[v * 4]);
    }
    auto flush = [&](int lo, int hi) {             // element range, widened to whole float4 (other CTAs hold zeros there)
      if (a.det_partials != nullptr) return;
      lo &= ~3;
      hi = (hi + 3) & ~3;
      if (hi > NPAR) hi = NPAR;
      for (int v = lo / 4 + tid; v < hi / 4; v += T) {
        const float4 q = *reinterpret_cast<const float4*>(&s.g[v * 4]);
        red_add_v4(gdst + v * 4, q.x, q.y, q.z, q.w);
      }
    };
    flush(W1 + cr * K::W1_PER, W1 + min(250, (cr + 1) * K::W1_PER));
    flush(B1, B1 + 10);                            // bias sums live in whichever CTA owns tap 0 of that channel (zeros elsewhere)
    flush(W2 + cr * K::W2_PER, W2 + (cr + 1) * K::W2_PER);
    flush(W3 + cr * K::FC1_PER * 320, W3 + min(50, (cr + 1) * K::FC1_PER) * 320);
    flush(B3 + cr * K::FC1_PER, B3 + min(50, (cr + 1) * K::FC1_PER));
    flush(W4 + cr * K::W4_PER, W4 + min(500, (cr + 1) * K::W4_PER));
    if (cr == 0) { flush(B2, B2 + 20); flush(B4, B4 + 10); }
  }
  if (tid == 0 && a.loss_acc != nullptr && cluster_id < a.B) {
    if (a.det_partials != nullptr && a.backward) {       // deterministic mode: the slot's padding carries the loss terms
      a.det_partials[(size_t)blockIdx.x * DET_STRIDE + NPAR] = cr == 0 ? s.loss_local * a.inv_bsz : 0.f;
      a.det_partials[(size_t)blockIdx.x * DET_STRIDE + NPAR + 1] = cr == 0 ? (float)s.correct_local : 0.f;
    } else if (cr == 0) {
      atomicAdd(a.loss_acc, s.loss_local * a.inv_bsz);
      atomicAdd(a.loss_acc + 1, (float)s.correct_local);
    }
  }
  cl.sync();                                       // no CTA exits while a peer may still address its shared memory
}

}  // namespace cnc

extern "C" {

// Returns 0 on success, cudaError otherwise.  `cluster` in {2, 4, 8}.
int b2_convnet_cluster_launch(const float* params, float* grads, const void* x, int x_u8, const long long* target,
                              float* loss_acc, float* out_logp, float* mask_out, const unsigned long long* step,
                              unsigned long long seed, long long sample_base, int B, int training, int backward,
                              float inv_bsz, float p_drop, int cluster, int max_clusters, long long grad_stride,
                              const float* aux, float* det_partials, cudaStream_t stream) {
  static bool configured = false;
  const size_t smem = sizeof(cnc::Smem);
  if (!configured) {
    cudaError_t e;
    if ((e = cudaFuncSetAttribute(cnc::convnet_cluster_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return (int)e;
    if ((e = cudaFuncSetAttribute(cnc::convnet_cluster_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return (int)e;
    if ((e = cudaFuncSetAttribute(cnc::convnet_cluster_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return (int)e;
    configured = true;
  }
  cn::Args a;
  a.params = params; a.grads = grads; a.x = x; a.target = target; a.loss_acc = loss_acc; a.out_logp = out_logp;
  a.mask_out = mask_out; a.step = step; a.seed = seed; a.sample_base = sample_base; a.B = B; a.x_u8 = x_u8;
  a.training = training; a.backward = backward; a.inv_bsz = inv_bsz; a.p_drop = p_drop;
  a.mean = 0.1307f; a.inv_std = 1.f / 0.3081f; a.grad_stride = grad_stride; a.aux = aux;
  a.det_partials = backward ? det_partials : nullptr;
  a.factors = nullptr; a.phase_ts = nullptr;
  int clusters = B;
  if (max_clusters > 0 && clusters > max_clusters) clusters = max_clusters;
  if (clusters < 1) clusters = 1;
  static const int pdl = [] { const char* e = getenv("B200DIST_PDL"); return (e == nullptr || e[0] != '0') ? 1 : 0; }();
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)(clusters * cluster));
  cfg.blockDim = dim3((unsigned)cnc::T);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 2 : 1;
  if (cluster == 2) return (int)cudaLaunchKernelEx(&cfg, cnc::convnet_cluster_kernel<2>, a);
  if (cluster == 4) return (int)cudaLaunchKernelEx(&cfg, cnc::convnet_cluster_kernel<4>, a);
  if (cluster == 8) return (int)cudaLaunchKernelEx(&cfg, cnc::convnet_cluster_kernel<8>, a);
  return (int)cudaErrorInvalidValue;
}

size_t b2_convnet_cluster_smem_bytes() { return sizeof(cnc::Smem); }

}  // extern "C"
