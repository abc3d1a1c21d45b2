// Fused MNIST-ConvNet training step for sm_90a: forward + loss + backward of the tutorial's `Net`
// (train_dist.py:53-71, nll_loss train_dist.py:120, backward :122) in ONE kernel.
//
// The reference runs ~35 library/ATen kernels per step (cuDNN convs, pools, relus, dropouts, cuBLAS
// linears, log_softmax, nll, and their backward twins) on [B,...] tensors that round-trip through
// HBM.  The network is per-sample independent and tiny (21,840 parameters, < 8 KB of activations per
// sample), so here one CTA carries a sample through the whole network and back with everything in
// shared memory / registers.  All weights (fc1.weight included) are staged once per CTA by 1-D bulk copies.
// Weight gradients are accumulated in shared memory and flushed once per CTA, except fc1.weight's, which each sample's fc1
// backward phase sends on by itself.  On one GPU (Args::factors) both leave with plain stores -- the accumulator to the CTA's
// slot, fc1's per-sample factors dh and p2 to a factor buffer -- and the optimizer kernel sums them in a fixed order
// (convnet_reduce.cuh).  Otherwise they are red.global.add.v4.f32-ed into the flat gradient bucket, the symmetric buffer the
// fused all-reduce + SGD kernel (sgd.cu) reads over NVSwitch.  HBM traffic per step is the input batch + one pass over the
// parameters; launches per step: 1 (+1 for the optimizer).
//
// Flat parameter layout (fp32, every tensor padded to 4 elements so all flushes are 16-byte vectors):
//   conv1.w 0 | conv1.b 252 | conv2.w 264 | conv2.b 5264 | fc1.w 5284 | fc1.b 21284 | fc2.w 21336 |
//   fc2.b 21836 | total 21848
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "common.cuh"
#include "tc_common.cuh"
#include "convnet_args.cuh"

namespace cn {

constexpr int T = 512;              // 16 warps per sample: the phases are latency-bound, so more warps per CTA

// The conv2 working set: fp32 weights in two layouts + split-K partial sums + the zero-padded conv2-output gradient
struct SimtBufs {
  float w2f[250 * 20];      // [ci][ky][kx][co]          forward: 4 output channels per float4
  float w2b[500 * 16];      // [co][ky][kx][half][8]     backward-data: 5 input channels per (half)
  float part[5 * 1440];     // conv2 partial sums [5][20][64] (5*1280 used) / dgrad partials [5][10][144] / S8b partials
  float dc2pad[DC_SIZE];      // conv2-output gradient, zero padded [20][16][16]
};

// fc1.weight has no slot in the shared gradient accumulator: S6 sends its per-sample gradient straight to global memory.
// The accumulator g holds the other parameters in flat order with the fc1.weight range cut out.
constexpr int NW3 = 16000, NG = NPAR - NW3;
__host__ __device__ constexpr int gslot(int i) { return i < W3 ? i : i - NW3; }   // flat index (not in fc1.weight) -> g

// The conv1-output gradient g1 is stored cell-major, [144 pooled cells][G1_CELL] with the 10 channels of a cell side by side:
// S8b reads the 10 channels of 3 cells per warp instruction, and S8a writes consecutive cells of one channel (odd stride:
// the 16 float2 of a half-warp land on distinct bank pairs).
constexpr int G1_CELL = 11;
// S7b splits the 20 output channels of the conv2 data gradient into 5 groups of 4, each summed into its own partial plane set
// of SimtBufs::part; S8a adds the 5 partials in group order.
constexpr int S7B_GROUPS = 5;
static_assert(3 * S7B_GROUPS <= T / 32 && 4 * S7B_GROUPS == 20, "S7b: three warps per group of four output channels");
// S8b: 8 warps take 6 of the 48 cell triples each; every (warp, cell slot) leaves one partial set of 26 sums x 10 channels.
constexpr int S8B_WARPS = 8, S8B_SET = 266;
static_assert(48 % S8B_WARPS == 0 && S8B_WARPS <= T / 32 && S8B_SET >= 260 && S8B_SET % 32 == 10, "S8b partition");
__host__ __device__ constexpr int g1_idx(int c, int cell) { return cell * G1_CELL + c; }

// Weights arrive by 1-D bulk copies straight from `params` / `aux`, so every staged array starts on a 16-byte boundary and
// arrays copied together are laid out as in `params`: [w1 | b1] = params[W1, W2), [w3 | b3 | w4 | b4] = params[W3, NPAR).
struct __align__(1024) Smem {
  SimtBufs u;
  alignas(16) float w1[252];
  float b1[12];
  alignas(16) float b2[20];
  alignas(16) float w3[NW3];  // fc1.weight [50][320], resident for the whole kernel (S3 and S6 read it)
  float b3[52];
  float w4[500];
  float b4[12];
  float x[784];
  float p1[P1_SIZE];        // relu(pool(conv1))  [10][12][12], padded strides (see convnet_args.cuh)
  float p2[320];            // relu(pool(drop(conv2)))  [20][4][4]
  float g2[320];            // gradient at the pooled conv2 argmax
  float2 g1[144 * G1_CELL]; // (gradient at the pooled conv1 argmax, input offset of that position as int bits), g1_idx
  float h[52];              // fc1 activation after relu+dropout
  float hm[52];             // fc1 backward mask (relu' * dropout scale)
  float dh[52];
  float dlog[12];
  float m2[20];             // dropout2d channel scale
  float rnd[72];            // uniforms: [0,20) dropout2d, [20,70) dropout
  alignas(16) float g[NG];  // per-CTA gradient accumulators (index with gslot)
  uint64_t bar[4];          // weight staging: [0] w1,b1,b2  [1] aux w2f  [2] w3,b3,w4,b4  [3] aux w2b
  int work_ctr;             // dynamic work distribution inside a phase (warp-granular)
  unsigned char a1[1440];   // conv1 pool argmax (0..3)
  unsigned char a2[320];    // conv2 pool argmax (0..3)
  float loss_local;
  int correct_local;
  int label;                // target of the current sample (loaded in S0 or, for a CTA's first sample, before pdl_wait)
};
static_assert(S7B_GROUPS * 1440 <= 5 * 1440 && 3 * S8B_WARPS * S8B_SET <= 5 * 1440, "S7b and S8b partials fit the scratch they reuse");
static_assert(sizeof(Smem) + 1024 <= 232448, "one CTA per SM: the launch asks for sizeof(Smem) + 1024 of the 227 KB opt-in");
static_assert(offsetof(Smem, b1) == offsetof(Smem, w1) + (B1 - W1) * 4 && offsetof(Smem, b3) == offsetof(Smem, w3) + (B3 - W3) * 4 &&
                  offsetof(Smem, w4) == offsetof(Smem, w3) + (W4 - W3) * 4 && offsetof(Smem, b4) == offsetof(Smem, w3) + (B4 - W3) * 4,
              "bulk-copied weight groups must be laid out as in params");
static_assert(W2 % 4 == 0 && B2 % 4 == 0 && W3 % 4 == 0 && NPAR % 4 == 0 && AUX_W2B % 4 == 0 && NG % 4 == 0,
              "bulk copies and float4 flushes need 16-byte offsets");

__global__ void __launch_bounds__(T, 1) convnet_step_kernel(Args a) {
  // the kernel has no static shared memory, so the dynamic window starts at offset 0 of the CTA's (1024-byte aligned)
  // shared space: addresses stay compile-time constants (a run-time round-up costs an extra add on every access)
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  const int tid = threadIdx.x;
  const float* __restrict__ P = a.params;
  const unsigned long long t_entry = a.phase_ts != nullptr ? b2::globaltimer() : 0ull;

  // sample b's image -> s.x (normalised), its label -> s.label
  auto load_input = [&](int b) {
    if (a.x_u8) {
      const uint4* xs = reinterpret_cast<const uint4*>(reinterpret_cast<const unsigned char*>(a.x) + (size_t)b * 784);
      if (tid < 49) {                              // 784 bytes = 49 x 16
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
    if (tid == 256) s.label = (int)__ldcg(a.target + b);
  };

  // ---------------------------------------------------------------- P0: stage weights, zero accumulators
  b2::pdl_launch_dependents();       // the all-reduce/SGD kernel may pre-launch; it parks in its own pdl_wait
  if (a.backward) {                  // everything that does not depend on the previous kernel happens before pdl_wait
    float4* g4 = reinterpret_cast<float4*>(s.g);
    for (int i = tid; i < NG / 4; i += T) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  // The CTA's first sample is loaded before pdl_wait, so its HBM latency overlaps the wait instead of following it.  The
  // kernel waited on is the optimizer kernel of the previous step: it writes parameters, momentum, aux, the step counter,
  // gradient buckets and loss terms, never a batch.  x and target arrive by copies ordered ahead of this launch (CUDA graph
  // nodes, or the executor's copy stream behind an event).  Callers that cannot promise that (x converted by the kernel
  // right before this one) leave input_ready off, and the sample is loaded in S0 like later ones.
  if (tid == 0) {                    // the staging barriers live in this CTA's shared memory: set them up while waiting
    for (int i = 0; i < 4; ++i) tc::mbar_init(&s.bar[i], 1);
    tc::mbar_fence_init();
  }
  const bool early = a.input_ready && (int)blockIdx.x < a.B;
  if (early) {
    load_input(blockIdx.x);
    if (a.backward)
      for (int i = tid; i < DC_SIZE / 4; i += T) reinterpret_cast<float4*>(s.u.dc2pad)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  b2::pdl_wait();                    // parameters / step counter written by the previous all-reduce+SGD kernel
  const unsigned long long t_waited = a.phase_ts != nullptr ? b2::globaltimer() : 0ull;
  // conv2.weight already in both smem layouts (written by sgd.cu): staged by bulk copies like the other weights
  const bool fast = a.aux != nullptr;
  if (tid == 0) {
    // One thread hands all weight staging to the TMA engine, in order of first use; each phase waits only for the group it
    // reads (S1: bar 0, S2: bar 1, S3: bar 2, S7b: bar 3), so the copies overlap the earlier phases.
    tc::fence_proxy_async_global();  // params / aux were written by the previous kernel through the generic proxy
    tc::mbar_expect_tx(&s.bar[0], (W2 - W1) * 4 + 80);
    tc::bulk_g2s(s.w1, P + W1, (W2 - W1) * 4, &s.bar[0]);                  // w1 | b1
    tc::bulk_g2s(s.b2, P + B2, 80, &s.bar[0]);
    if (fast) {
      tc::mbar_expect_tx(&s.bar[1], AUX_W2B * 4);
      tc::bulk_g2s(s.u.w2f, a.aux + AUX_W2F, AUX_W2B * 4, &s.bar[1]);
    }
    tc::mbar_expect_tx(&s.bar[2], (NPAR - W3) * 4);
    tc::bulk_g2s(s.w3, P + W3, (NPAR - W3) * 4, &s.bar[2]);              // w3 | b3 | w4 | b4
    if (fast) {
      tc::mbar_expect_tx(&s.bar[3], (AUX_TOTAL - AUX_W2B) * 4);
      tc::bulk_g2s(s.u.w2b, a.aux + AUX_W2B, (AUX_TOTAL - AUX_W2B) * 4, &s.bar[3]);
    }
  }
  {
    // without aux: conv2.weight is scattered into its smem layouts from registers (all loads in flight before the first store)
    const float4* __restrict__ P4w2 = reinterpret_cast<const float4*>(P + W2);   // 1250 float4, 16B aligned
    float4 v[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int i4 = tid + k * T;
      v[k] = (!fast && i4 < 1250) ? __ldg(P4w2 + i4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int i4 = tid + k * T;
      if (!fast && i4 < 1250) {
        const float w[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {             // conv2.weight [co][ci][ky][kx]
          const int i = i4 * 4 + e;
          const int co = i / 250, r = i % 250, ci = r / 25, kk = r % 25;
          s.u.w2f[(ci * 25 + kk) * 20 + co] = w[e];
          s.u.w2b[((co * 25 + kk) * 2 + ci / 5) * 8 + ci % 5] = w[e];
        }
      }
    }
  }
  if (tid == 0) { s.loss_local = 0.f; s.correct_local = 0; }
  const unsigned long long step = a.step ? *a.step : 0ull;
  // correctly rounded 1 / (1 - p): --use_fast_math would turn the division into the approximate MUFU reciprocal, 1 ulp off
  // for some p (0.9), and the scale would differ from the one the host and the other engines apply
  const float keep_scale = __frcp_rn(1.f - a.p_drop);
  // this step's gradient bucket (double-buffered: see sgd.cu); fc1.weight's share goes there from S6, the rest in the flush
  float* const gdst = a.backward ? a.grads + (size_t)(step & 1ull) * (size_t)a.grad_stride : nullptr;
  // The barrier that ends S0 publishes the mbarrier initialisation and the scattered conv2.weight before any phase reads
  // them, so the RNG of S0 need not wait here for thread 0's copy issue.
  auto stamp = [&](int k) {          // opt-in phase timestamps (bench/step_phases.py); call after a barrier
    if (a.phase_ts != nullptr && tid == 0) b2::ts_put(a.phase_ts, step, (int)blockIdx.x, k, b2::globaltimer());
  };
  if (a.phase_ts != nullptr && tid == 0) {
    b2::ts_put(a.phase_ts, step, (int)blockIdx.x, b2::TS_ENTRY, t_entry);
    b2::ts_put(a.phase_ts, step, (int)blockIdx.x, b2::TS_WAITED, t_waited);
  }

  for (int b = blockIdx.x; b < a.B; b += gridDim.x) {
    // -------------------------------------------------------------- S0: input, RNG, clear scratch
    const bool loaded = early && b == (int)blockIdx.x;   // first sample: input and cleared dc2pad are in place already
    if (!loaded) load_input(b);
    if (tid >= 256 && tid < 274) {
      const int q = tid - 256;
      uint4 r = b2::Philox::gen(a.seed, (unsigned long long)(a.sample_base + b), step * 32ull + q);
      const float k = 2.3283064365386963e-10f;   // 2^-32
      s.rnd[q * 4 + 0] = r.x * k; s.rnd[q * 4 + 1] = r.y * k;
      s.rnd[q * 4 + 2] = r.z * k; s.rnd[q * 4 + 3] = r.w * k;
    }
    if (a.backward && !loaded)
      for (int i = tid; i < DC_SIZE / 4; i += T) reinterpret_cast<float4*>(s.u.dc2pad)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    stamp(b2::TS_S0);

    // -------------------------------------------------------------- S1: conv1 -> maxpool2 -> relu
    tc::mbar_wait(&s.bar[0], 0);                   // w1, b1, b2 (after the first sample: returns at once)
    if (tid < 480) {                               // 48 threads per channel, 3 pooled cells each: the 25 weights stay in registers
      const int c = tid / 48;
      float w[25];
#pragma unroll
      for (int k = 0; k < 25; ++k) w[k] = s.w1[c * 25 + k];
      const float bias = s.b1[c];
#pragma unroll 1
      for (int r = tid - c * 48; r < 144; r += 48) {
        const int o = c * 144 + r, py = r / 12, px = r % 12;
        float patch[6][6];
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
          for (int j = 0; j < 3; ++j) {              // 8-byte aligned pairs: 18 LDS.64 instead of 36 LDS.32
            const float2 q = *reinterpret_cast<const float2*>(&s.x[(2 * py + i) * 28 + 2 * px + 2 * j]);
            patch[i][2 * j] = q.x; patch[i][2 * j + 1] = q.y;
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
        float m = a00; int arg = 0;
        if (a01 > m) { m = a01; arg = 1; }
        if (a10 > m) { m = a10; arg = 2; }
        if (a11 > m) { m = a11; arg = 3; }
        s.p1[p1_idx(c, py, px)] = fmaxf(m, 0.f);
        s.a1[o] = (unsigned char)arg;
      }
    }
    if (tid < 20)
      s.m2[tid] = a.training ? (s.rnd[tid] >= a.p_drop ? keep_scale : 0.f) : 1.f;
    __syncthreads();
    stamp(b2::TS_S1);

    // -------------------------------------------------------------- S2: conv2 (K split 5)
    if (fast) tc::mbar_wait(&s.bar[1], 0);         // w2f
    if (tid < 400) {
      const int cell = tid & 15, cg = (tid >> 4) % 5, ks = tid / 80;
      const int py = cell >> 2, px = cell & 3;
      const int ci0 = 2 * ks, ci1 = 2 * ks + 2;
      float acc[4][4];
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[p][c] = 0.f;
      for (int ci = ci0; ci < ci1; ++ci) {
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
            const float4 w = *reinterpret_cast<const float4*>(&s.u.w2f[((ci * 5 + ky) * 5 + kx) * 20 + cg * 4]);
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
      }
      // part[ks][co][cell][pos]  (pos = dy*2+dx inside the pool window)
#pragma unroll
      for (int c = 0; c < 4; ++c)
        *reinterpret_cast<float4*>(&s.u.part[ks * 1440 + ((cg * 4 + c) * 16 + cell) * 4]) =
            make_float4(acc[0][c], acc[1][c], acc[2][c], acc[3][c]);
    }
    __syncthreads();

    // -------------------------------------------------------------- S2b: +bias, dropout2d, maxpool2, relu
    for (int o = tid; o < 320; o += T) {
      const int co = o >> 4;
      float4 q = *reinterpret_cast<const float4*>(&s.u.part[o * 4]);
#pragma unroll
      for (int ks = 1; ks < 5; ++ks) {
        const float4 t = *reinterpret_cast<const float4*>(&s.u.part[ks * 1440 + o * 4]);
        q.x += t.x; q.y += t.y; q.z += t.z; q.w += t.w;
      }
      const float bias = s.b2[co], sc = s.m2[co];
      const float v0 = (q.x + bias) * sc, v1 = (q.y + bias) * sc, v2 = (q.z + bias) * sc, v3 = (q.w + bias) * sc;
      float m = v0; int arg = 0;
      if (v1 > m) { m = v1; arg = 1; }
      if (v2 > m) { m = v2; arg = 2; }
      if (v3 > m) { m = v3; arg = 3; }
      s.p2[o] = fmaxf(m, 0.f);
      s.a2[o] = (unsigned char)arg;
    }
    __syncthreads();
    stamp(b2::TS_S2);

    // -------------------------------------------------------------- S3: fc1 + relu + dropout
    tc::mbar_wait(&s.bar[2], 0);                   // w3, b3, w4, b4
    {
      const int j = tid >> 3, l8 = tid & 7;
      float sum = 0.f;
      if (j < 50) {
        const float4* wrow = reinterpret_cast<const float4*>(s.w3 + j * 320);   // 4 rows x 128 B per warp: no conflicts
#pragma unroll
        for (int k = 0; k < 10; ++k) {
          const float4 w = wrow[l8 + 8 * k];
          const float4 v = *reinterpret_cast<const float4*>(&s.p2[(l8 + 8 * k) * 4]);
          sum = fmaf(w.x, v.x, sum); sum = fmaf(w.y, v.y, sum);
          sum = fmaf(w.z, v.z, sum); sum = fmaf(w.w, v.w, sum);
        }
      }
      sum += __shfl_xor_sync(0xffffffffu, sum, 4);
      sum += __shfl_xor_sync(0xffffffffu, sum, 2);
      sum += __shfl_xor_sync(0xffffffffu, sum, 1);
      if (j < 50 && l8 == 0) {
        const float pre = sum + s.b3[j];
        const float dm = a.training ? (s.rnd[20 + j] >= a.p_drop ? keep_scale : 0.f) : 1.f;
        s.h[j] = fmaxf(pre, 0.f) * dm;
        s.hm[j] = pre > 0.f ? dm : 0.f;
      }
    }
    __syncthreads();

    // -------------------------------------------------------------- S4: fc2 + log_softmax + nll
    if (tid < 32) {
      const int y = s.label;
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
        if (a.out_logp) a.out_logp[(size_t)b * 10 + tid] = logp;
        s.dlog[tid] = (e / se - (tid == (int)y ? 1.f : 0.f)) * a.inv_bsz;
        if (tid == (int)y) s.loss_local += -logp;
      }
      if (tid == 0 && am == (int)y) s.correct_local += 1;
    }
    if (a.mask_out) {
      if (tid < 20) a.mask_out[(size_t)b * 70 + tid] = s.m2[tid];
      else if (tid < 70) a.mask_out[(size_t)b * 70 + tid] =
          a.training ? (s.rnd[tid] >= a.p_drop ? keep_scale : 0.f) : 1.f;
    }
    __syncthreads();
    stamp(b2::TS_S4);
    if (!a.backward) continue;

    // -------------------------------------------------------------- S5: fc2 backward
    for (int e = tid; e < 500; e += T) s.g[gslot(W4) + e] += s.dlog[e / 50] * s.h[e % 50];
    if (tid < 10) s.g[gslot(B4) + tid] += s.dlog[tid];
    if (tid >= 64 && tid < 114) {
      const int i = tid - 64;
      float d = 0.f;
#pragma unroll
      for (int k = 0; k < 10; ++k) d = fmaf(s.w4[k * 50 + i], s.dlog[k], d);
      s.dh[i] = d * s.hm[i];
    }
    __syncthreads();

    // -------------------------------------------------------------- S6: fc1 backward
    {
      // data gradient first: S7 waits for it, while the atomics below only have to be issued
      if (tid >= 320 && tid < 370) s.g[gslot(B3) + tid - 320] += s.dh[tid - 320];
      if (tid == 511) s.work_ctr = 0;
      for (int o = tid; o < 320; o += T) {
        float d = 0.f;
#pragma unroll 10
        for (int jj = 0; jj < 50; ++jj) d = fmaf(s.w3[jj * 320 + o], s.dh[jj], d);
        const int co = o >> 4, cell = o & 15, arg = s.a2[o];
        const float gv = s.p2[o] > 0.f ? d * s.m2[co] : 0.f;
        s.g2[o] = gv;
        const int y = 2 * (cell >> 2) + (arg >> 1), x = 2 * (cell & 3) + (arg & 1);
        s.u.dc2pad[co * DC_PLANE + (y + 4) * DC_ROW + (x + 4)] = gv;
      }
      // fc1.weight gradient dh (x) p2 of this sample goes straight to global memory: as its two factors (370 floats, stored
      // by threads that are idle in this phase; the reduction of convnet_reduce.cuh forms the sum over samples), or as the
      // product, 4 consecutive inputs per thread-iteration, into this CTA's slot (det_partials) or red.add-ed into the bucket.
      const float4* p24 = reinterpret_cast<const float4*>(s.p2);
      if (a.factors != nullptr) {
        float* f = a.factors + (size_t)b * FAC_STRIDE;
        if (tid >= 370 && tid < 420) f[tid - 370] = s.dh[tid - 370];
        else if (tid >= 420 && tid < 500) reinterpret_cast<float4*>(f + FAC_P2)[tid - 420] = p24[tid - 420];
      } else if (a.det_partials != nullptr) {
        float4* slot = reinterpret_cast<float4*>(a.det_partials + (size_t)blockIdx.x * DET_STRIDE + W3);
        const bool first = b == (int)blockIdx.x;  // later samples of the same CTA add to what this thread stored before
        for (int e4 = tid; e4 < 4000; e4 += T) {
          const int j = e4 / 80, i4 = e4 - j * 80;
          const float d = s.dh[j];
          const float4 pv = p24[i4];
          float4 gv = first ? make_float4(0.f, 0.f, 0.f, 0.f) : slot[e4];
          gv.x = fmaf(d, pv.x, gv.x); gv.y = fmaf(d, pv.y, gv.y); gv.z = fmaf(d, pv.z, gv.z); gv.w = fmaf(d, pv.w, gv.w);
          slot[e4] = gv;
        }
      } else {
        for (int e4 = tid; e4 < 4000; e4 += T) {
          const int j = e4 / 80, i4 = e4 - j * 80;
          const float d = s.dh[j];
          const float4 pv = p24[i4];
          red_add_v4(gdst + W3 + e4 * 4, d * pv.x, d * pv.y, d * pv.z, d * pv.w);
        }
      }
    }
    __syncthreads();
    stamp(b2::TS_S6);

    // -------------------------------------------------------------- S7a: conv2 weight/bias gradient (sparse)
    // Work items are handed out 32 at a time per warp from a shared counter, so the warps that had no (or a short)
    // S7b tile start here immediately and the phase ends balanced.  item < 1000: (co, ci, ky) = 5 taps x 16 pooled
    // cells; item 1000..1019: bias gradient of channel item-1000.
    auto s7a = [&]() {
      for (;;) {
        int base = 0;
        if ((tid & 31) == 0) base = atomicAdd(&s.work_ctr, 32);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= 1020) break;
        const int item = base + (tid & 31);
        if (item < 1000) {
          const int co = item / 50, r = item - co * 50, ci = r / 5, ky = r - ci * 5;
          float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
          for (int cell = 0; cell < 16; ++cell) {
            const float gv = s.g2[co * 16 + cell];
            if (gv != 0.f) {
              const int arg = s.a2[co * 16 + cell];
              const int ay = 2 * (cell >> 2) + (arg >> 1), ax = 2 * (cell & 3) + (arg & 1);
              const float* src = &s.p1[p1_idx(ci, ay + ky, ax)];
#pragma unroll
              for (int kx = 0; kx < 5; ++kx) acc[kx] = fmaf(gv, src[kx], acc[kx]);
            }
          }
          float* dst = &s.g[gslot(W2) + co * 250 + ci * 25 + ky * 5];
#pragma unroll
          for (int kx = 0; kx < 5; ++kx) dst[kx] += acc[kx];
        } else if (item < 1020) {
          const int co = item - 1000;
          float d = 0.f;
#pragma unroll
          for (int cell = 0; cell < 16; ++cell) d += s.g2[co * 16 + cell];
          s.g[gslot(B2) + co] += d;
        }
      }
    };
    // -------------------------------------------------------------- S7b: conv2 data gradient
    if (fast) tc::mbar_wait(&s.bar[3], 0);         // w2b
    // Warp-uniform channel ranges: warps 3g .. 3g+2 take output channels 4g .. 4g+3 (a Dropout2d skip skips the whole warp)
    // and together cover 12 rows x 4 column triples x 2 input-channel halves; lane = (half, row 4k + r, column triple q).
    // The 16 (row, triple) dc2pad addresses of a load fall on distinct banks (row stride 20, triple stride 3), and the two
    // halves read the same words.  Warp 15 and the warps whose channels are dropped go on to the S7a items.
    if (tid < 32 * 3 * S7B_GROUPS) {
      const int warp = tid >> 5, lane = tid & 31, cg = warp / 3;
      const int half = lane >> 4, y = 4 * (warp - 3 * cg) + ((lane >> 2) & 3), x0 = 3 * (lane & 3);
      float acc[3][5];
#pragma unroll
      for (int p = 0; p < 3; ++p)
#pragma unroll
        for (int c = 0; c < 5; ++c) acc[p][c] = 0.f;
      for (int co = 4 * cg; co < 4 * cg + 4; ++co) {
        if (s.m2[co] == 0.f) continue;            // channel dropped by Dropout2d: gradient plane is zero (warp-uniform)
        float patch[5][7];
        const float* src = &s.u.dc2pad[co * DC_PLANE + y * DC_ROW + x0];
#pragma unroll
        for (int i = 0; i < 5; ++i)
#pragma unroll
          for (int jx = 0; jx < 7; ++jx) patch[i][jx] = src[i * DC_ROW + jx];
#pragma unroll
        for (int ky = 0; ky < 5; ++ky)
#pragma unroll
          for (int kx = 0; kx < 5; ++kx) {
            const float* wp = &s.u.w2b[((co * 25 + ky * 5 + kx) * 2 + half) * 8];
            const float4 w = *reinterpret_cast<const float4*>(wp);
            const float w4 = wp[4];
#pragma unroll
            for (int p = 0; p < 3; ++p) {
              const float d = patch[4 - ky][4 - kx + p];
              acc[p][0] = fmaf(w.x, d, acc[p][0]); acc[p][1] = fmaf(w.y, d, acc[p][1]);
              acc[p][2] = fmaf(w.z, d, acc[p][2]); acc[p][3] = fmaf(w.w, d, acc[p][3]); acc[p][4] = fmaf(w4, d, acc[p][4]);
            }
          }
      }
#pragma unroll
      for (int c = 0; c < 5; ++c) {
        float* dst = &s.u.part[cg * 1440 + (half * 5 + c) * 144 + y * 12 + x0];
        dst[0] = acc[0][c]; dst[1] = acc[1][c]; dst[2] = acc[2][c];
      }
    }
    s7a();
    __syncthreads();

    // -------------------------------------------------------------- S8a: through relu+pool of conv1
    for (int o = tid; o < 1440; o += T) {
      float d = 0.f;
#pragma unroll
      for (int cg = 0; cg < S7B_GROUPS; ++cg) d += s.u.part[cg * 1440 + o];
      const int cell = o % 144, arg = s.a1[o];
      const int off = (2 * (cell / 12) + (arg >> 1)) * 28 + 2 * (cell % 12) + (arg & 1);
      s.g1[g1_idx(o / 144, cell)] = make_float2(s.p1[p1_of(o)] > 0.f ? d : 0.f, __int_as_float(off));
    }
    __syncthreads();
    stamp(b2::TS_S8A);

    // -------------------------------------------------------------- S8b: conv1 weight/bias gradient (sparse)
    // Lanes over cells: lane (j, c) of warps 0-7 takes channel c of the pooled cells (py, px0 + 4j), py = t / 4, px0 = t % 4,
    // for the 6 triples t = w, w + 8, ..., w + 40, and gathers the 5x5 input window at each cell's argmax into 25 register
    // sums (+ the bias sum).  The addresses of one load differ by 8 banks between the three cells and by an argmax step (0,
    // 1, 28 or 29 words) inside a cell: all 30 lanes hit distinct banks or share a word.  The 24 partial sets (one per warp
    // and j) go to shared memory and are added in set order.
    {
      float* const red = s.u.part;   // [24 sets][S8B_SET], dead after S8a
      const int lane = tid & 31, warp = tid >> 5, j = lane / 10, c = lane - j * 10;
      if (warp < S8B_WARPS) {
        float acc[26];
#pragma unroll
        for (int k = 0; k < 26; ++k) acc[k] = 0.f;
        if (j < 3) {
#pragma unroll 2
          for (int t = warp; t < 48; t += S8B_WARPS) {
            const float2 q = s.g1[g1_idx(c, (t >> 2) * 12 + (t & 3) + 4 * j)];
            const float* src = &s.x[__float_as_int(q.y)];
#pragma unroll
            for (int k = 0; k < 25; ++k) acc[k] = fmaf(q.x, src[(k / 5) * 28 + k % 5], acc[k]);
            acc[25] += q.x;
          }
          float* dst = red + (warp * 3 + j) * S8B_SET + c;   // set stride = 10 (mod 32): the 30 lanes store to 30 banks
#pragma unroll
          for (int k = 0; k < 26; ++k) dst[k * 10] = acc[k];
        }
      }
      __syncthreads();
      if (tid < 260) {
        float d = 0.f;
#pragma unroll
        for (int set = 0; set < 3 * S8B_WARPS; ++set) d += red[set * S8B_SET + tid];
        const int k = tid / 10, ch = tid - k * 10;
        if (k < 25) s.g[gslot(W1) + ch * 25 + k] += d;
        else s.g[gslot(B1) + ch] += d;
      }
    }
    __syncthreads();
    stamp(b2::TS_S8B);
  }

  // ------------------------------------------------------------------ flush (everything but fc1.weight, which S6 sent already)
  if (a.backward && blockIdx.x < a.B) {
    if (a.det_partials != nullptr) {        // deterministic mode: a private slot per CTA, summed in CTA order afterwards
      float* slot = a.det_partials + (size_t)blockIdx.x * DET_STRIDE;
      for (int v = tid; v < NG / 4; v += T) {
        const int i = v * 4 < W3 ? v * 4 : v * 4 + NW3;   // inverse of gslot
        *reinterpret_cast<float4*>(slot + i) = *reinterpret_cast<const float4*>(&s.g[v * 4]);
      }
    } else {
      for (int v = tid; v < NG / 4; v += T) {
        const int i = v * 4 < W3 ? v * 4 : v * 4 + NW3;
        const float4 q = *reinterpret_cast<const float4*>(&s.g[v * 4]);
        red_add_v4(gdst + i, q.x, q.y, q.z, q.w);
      }
    }
  }
  if (a.phase_ts != nullptr) {
    __syncthreads();
    stamp(b2::TS_FLUSHED);
  }
  // no bulk copy may still be writing this CTA's shared memory when it exits (groups no phase waited for: forward-only runs,
  // a CTA without samples)
  if (tid == 0) {
    tc::mbar_wait(&s.bar[0], 0);
    tc::mbar_wait(&s.bar[2], 0);
    if (fast) { tc::mbar_wait(&s.bar[1], 0); tc::mbar_wait(&s.bar[3], 0); }
  }
  if (tid == 0 && a.loss_acc != nullptr && blockIdx.x < a.B) {
    if (a.det_partials != nullptr && a.backward) {       // deterministic mode: the slot's padding carries this CTA's loss terms
      a.det_partials[(size_t)blockIdx.x * DET_STRIDE + NPAR] = s.loss_local * a.inv_bsz;
      a.det_partials[(size_t)blockIdx.x * DET_STRIDE + NPAR + 1] = (float)s.correct_local;
    } else {
      atomicAdd(a.loss_acc, s.loss_local * a.inv_bsz);
      atomicAdd(a.loss_acc + 1, (float)s.correct_local);
    }
  }
  stamp(b2::TS_EXIT);
}

}  // namespace cn

extern "C" {

unsigned long long* b2_phase_ts();   // sgd.cu

size_t b2_convnet_smem_bytes() { return sizeof(cn::Smem) + 1024; }
int b2_convnet_npar() { return cn::NPAR; }

int b2_convnet_step_launch(const float* params, float* grads, const void* x, int x_u8, const long long* target,
                           float* loss_acc, float* out_logp, float* mask_out, const unsigned long long* step,
                           unsigned long long seed, long long sample_base, int B, int training, int backward,
                           float inv_bsz, float p_drop, int max_ctas, long long grad_stride, const float* aux,
                           float* det_partials, float* factors, int input_ready, cudaStream_t stream) {
  static bool configured = false;
  const size_t smem = sizeof(cn::Smem) + 1024;
  if (!configured) {
    const cudaError_t e = cudaFuncSetAttribute(cn::convnet_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  cn::Args a;
  a.params = params; a.grads = grads; a.x = x; a.target = target; a.loss_acc = loss_acc; a.out_logp = out_logp;
  a.mask_out = mask_out; a.step = step; a.seed = seed; a.sample_base = sample_base; a.B = B; a.x_u8 = x_u8;
  a.training = training; a.backward = backward; a.inv_bsz = inv_bsz; a.p_drop = p_drop;
  a.mean = 0.1307f; a.inv_std = 1.f / 0.3081f; a.grad_stride = grad_stride; a.aux = aux;
  a.det_partials = backward ? det_partials : nullptr;
  a.factors = (backward && det_partials != nullptr) ? factors : nullptr;
  a.phase_ts = b2_phase_ts();
  a.input_ready = input_ready;
  int grid = B;
  if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
  if (grid < 1) grid = 1;
  static const int pdl = [] { const char* e = getenv("B200DIST_PDL"); return (e == nullptr || e[0] != '0') ? 1 : 0; }();
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3((unsigned)cn::T);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return (int)cudaLaunchKernelEx(&cfg, cn::convnet_step_kernel, a);
}

}  // extern "C"
