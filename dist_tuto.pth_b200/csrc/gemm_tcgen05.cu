// bf16 GEMM on the Hopper tensor cores (sm_90a), hand-written:
//   C[M,N] = A[M,K] * B[N,K]^T (+ bias[N]) (ReLU)      A, B bf16 K-contiguous; fp32 accumulation in registers
//
// This is the linear-layer engine of the framework (fc1/fc2 of the tutorial Net at large batch,
// ResNet-18's classifier, and the implicit-GEMM convolutions built on top of it):
//   warpgroup 0     : TMA producer  -- one thread issues cp.async.bulk.tensor.2d (128B-swizzled tiles) into a smem ring
//   warpgroups 1, 2 : consumers     -- wgmma.mma_async m64nBNk16 on rows 0..63 / 64..127 of the 128-row tile, then
//                                      bias/ReLU -> bf16/fp32 -> global stores straight from the accumulator registers
// Large GEMMs (N >= 192, K >= 2048, at least one wave of tiles) take a persistent kernel with 128x256 tiles instead.
// Synchronisation is mbarrier-only (full/empty per stage).  Ragged M/N/K edges are handled by TMA out-of-bounds zero fill
// and predicated stores.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <string>

#include "tc_common.cuh"

namespace gemm {

constexpr int BM = 128, BK = 64;
// stages: the TMA ring runs up to STAGES k-blocks ahead of the MMAs
template <int BN> struct Cfg { static constexpr int STAGES = BN >= 128 ? 3 : 4; };
constexpr int kThreads = 384;

// One warpgroup's share (64 rows) of a 128 x BN tile: K loop over the smem ring.  The MMAs of k-block kb run while the
// warpgroup waits for k-block kb+1; a stage is released once the MMAs reading it have completed.  `it` is the running
// k-block counter that selects stage and phase (it continues across the tiles of a persistent CTA).
template <int BN, int STAGES>
__device__ __forceinline__ uint32_t mma_tile(float* d, const uint8_t* a_ring, const uint8_t* b_ring, uint64_t* full,
                                             uint64_t* empty, int half, int num_kb, uint32_t it) {
  constexpr uint32_t kABytes = BM * BK * 2, kBBytes = BN * BK * 2;
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
  for (int kb = 0; kb < num_kb; ++kb, ++it) {
    const uint32_t st = it % STAGES;
    tc::mbar_wait(&full[st], (it / STAGES) & 1);
    const uint32_t a_addr = tc::smem_u32(a_ring) + st * kABytes + half * 64 * 128, b_addr = tc::smem_u32(b_ring) + st * kBBytes;
    tc::wg_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)                    // +16 bf16 = 32 B inside the 128 B swizzle row
      tc::mma<BN>(d, tc::smem_desc_sw128(a_addr + k * 32), tc::smem_desc_sw128(b_addr + k * 32), 1u);
    tc::wg_commit();
    tc::wg_wait_1();                                     // k-block kb-1 done: its stage is free
    if (kb > 0) tc::mbar_arrive(&empty[(it - 1) % STAGES]);
  }
  tc::wg_wait_all();
  tc::acc_fence<BN / 2>(d);
  tc::mbar_arrive(&empty[(it - 1) % STAGES]);
  return it;
}

// bias / ReLU / bf16 or fp32 stores straight from the accumulator registers of one warpgroup (rows row0..row0+63)
template <int BN>
__device__ __forceinline__ void store_tile(const float* d, int t, int row0, int n0, void* __restrict__ c,
                                           const float* __restrict__ bias, int M, int N, int relu, int out_bf16) {
  const bool pairs = (N % 2) == 0;
#pragma unroll
  for (int i = 0; i < BN / 2; i += 2) {
    const int row = row0 + tc::acc_row(t, i), col = n0 + tc::acc_col(t, i);
    if (row >= M || col >= N) continue;
    float v0 = d[i], v1 = d[i + 1];
    if (bias != nullptr) {
      v0 += __ldg(bias + col);
      if (col + 1 < N) v1 += __ldg(bias + col + 1);
    }
    if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
    if (out_bf16) {
      __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(c) + (size_t)row * N + col;
      if (pairs) *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(v0, v1);
      else { dst[0] = __float2bfloat16(v0); if (col + 1 < N) dst[1] = __float2bfloat16(v1); }
    } else {
      float* dst = reinterpret_cast<float*>(c) + (size_t)row * N + col;
      if (pairs) *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
      else { dst[0] = v0; if (col + 1 < N) dst[1] = v1; }
    }
  }
}

template <int BN, int STAGES>
struct SmemLayout {
  alignas(1024) uint8_t a[STAGES][BM * BK * 2];
  alignas(1024) uint8_t b[STAGES][BN * BK * 2];
  alignas(8) uint64_t full[STAGES];
  alignas(8) uint64_t empty[STAGES];
};

template <int BN, int STAGES>
__device__ __forceinline__ void init_ring(SmemLayout<BN, STAGES>& s, const CUtensorMap* map_a, const CUtensorMap* map_b) {
  if (threadIdx.x == 0) {
    tc::prefetch_tmap(map_a);
    tc::prefetch_tmap(map_b);
    for (int i = 0; i < STAGES; ++i) { tc::mbar_init(&s.full[i], 1); tc::mbar_init(&s.empty[i], 2 * 128); }
    tc::mbar_fence_init();
  }
  __syncthreads();
}

template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, void* __restrict__ c,
                 const float* __restrict__ bias, int M, int N, int K, int relu, int out_bf16) {
  constexpr int STAGES = Cfg<BN>::STAGES;
  using Smem = SmemLayout<BN, STAGES>;
  extern __shared__ uint8_t smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int num_kb = (K + BK - 1) / BK;
  init_ring(s, &map_a, &map_b);

  if (wg == 0) {
    // ======================================================== TMA producer
    if (t == 0) {
      for (int kb = 0; kb < num_kb; ++kb) {
        const int st = kb % STAGES;
        tc::mbar_wait(&s.empty[st], ((kb / STAGES) & 1) ^ 1);   // first pass: parity 1 passes on a fresh barrier
        tc::mbar_expect_tx(&s.full[st], (BM + BN) * BK * 2);
        tc::tma_load_2d(s.a[st], &map_a, &s.full[st], kb * BK, m0);
        tc::tma_load_2d(s.b[st], &map_b, &s.full[st], kb * BK, n0);
      }
    }
    return;
  }
  // ========================================================== consumers: warpgroup 1 -> rows 0..63, 2 -> rows 64..127
  const int half = wg - 1;
  float d[BN / 2];
  mma_tile<BN, STAGES>(d, &s.a[0][0], &s.b[0][0], s.full, s.empty, half, num_kb, 0u);
  store_tile<BN>(d, t, m0 + half * 64, n0, c, bias, M, N, relu, out_bf16);
}

// ------------------------------------------------------------------------------------------ persistent 128x256 kernel
// Large GEMMs: one CTA per SM loops over output tiles; 128x256 tiles halve the operand bytes per FLOP relative to 128x128,
// and the producer keeps the 4-stage ring filled with the next tile's k-blocks while the consumers run the epilogue of
// the current one.  Each consumer warpgroup holds a 64x256 fp32 accumulator (128 registers per thread): the producer
// warpgroup hands most of its register budget to them (setmaxnreg).
constexpr int PBN = 256, PSTAGES = 4;
using PSmem = SmemLayout<PBN, PSTAGES>;

__global__ void __launch_bounds__(kThreads, 1)
gemm_bf16_persistent_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                            void* __restrict__ c, const float* __restrict__ bias, int M, int N, int K, int relu, int out_bf16) {
  extern __shared__ uint8_t smem_raw[];
  PSmem& s = *reinterpret_cast<PSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int mt = (M + BM - 1) / BM, nt = (N + PBN - 1) / PBN, tiles = mt * nt;
  const int num_kb = (K + BK - 1) / BK;
  init_ring(s, &map_a, &map_b);

  if (wg == 0) {
    tc::regs_dec<40>();
    if (t == 0) {
      uint32_t it = 0;                                          // global k-block counter -> stage / phase
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int m0 = (tile % mt) * BM, n0 = (tile / mt) * PBN;   // consecutive CTAs share the B (N) panel
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int st = it % PSTAGES;
          tc::mbar_wait(&s.empty[st], ((it / PSTAGES) & 1) ^ 1);
          tc::mbar_expect_tx(&s.full[st], (BM + PBN) * BK * 2);
          tc::tma_load_2d(s.a[st], &map_a, &s.full[st], kb * BK, m0);
          tc::tma_load_2d(s.b[st], &map_b, &s.full[st], kb * BK, n0);
        }
      }
    }
    return;
  }
  tc::regs_inc<232>();
  const int half = wg - 1;
  uint32_t it = 0;
  float d[PBN / 2];
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int m0 = (tile % mt) * BM, n0 = (tile / mt) * PBN;
    it = mma_tile<PBN, PSTAGES>(d, &s.a[0][0], &s.b[0][0], s.full, s.empty, half, num_kb, it);
    store_tile<PBN>(d, t, m0 + half * 64, n0, c, bias, M, N, relu, out_bf16);
  }
}

// ------------------------------------------------------------------------------------------ host side
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

// 2-D bf16 row-major [rows, k] tensor, box = [box_rows, 64], 128B swizzle, OOB -> zero
bool make_map(CUtensorMap* map, const void* ptr, int rows, int k, int box_rows) {
  EncodeFn enc = get_encode();
  if (!enc) { g_err = "cuTensorMapEncodeTiled not available (no CUDA driver?)"; return false; }
  cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)k * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { g_err = "cuTensorMapEncodeTiled failed: " + std::to_string((int)r); return false; }
  return true;
}

template <int BN>
int launch(const void* a, const void* b, void* c, const float* bias, int M, int N, int K, int relu, int out_bf16,
           cudaStream_t stream) {
  CUtensorMap ma, mb;
  if (!make_map(&ma, a, M, K, BM) || !make_map(&mb, b, N, K, BN)) return -1;
  const size_t smem = sizeof(SmemLayout<BN, Cfg<BN>::STAGES>) + 1024;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { g_err = std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e); return -2; }
    configured = true;
  }
  dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN);
  gemm_bf16_kernel<BN><<<grid, kThreads, smem, stream>>>(ma, mb, c, bias, M, N, K, relu, out_bf16);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { g_err = std::string("launch: ") + cudaGetErrorString(e); return -3; }
  return 0;
}

int launch_persistent(const void* a, const void* b, void* c, const float* bias, int M, int N, int K, int relu, int out_bf16,
                      cudaStream_t stream) {
  CUtensorMap ma, mb;
  if (!make_map(&ma, a, M, K, BM) || !make_map(&mb, b, N, K, PBN)) return -1;
  const size_t smem = sizeof(PSmem) + 1024;
  static int sms = 0;
  if (sms == 0) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_persistent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { g_err = std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e); return -2; }
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  const int tiles = ((M + BM - 1) / BM) * ((N + PBN - 1) / PBN);
  const int grid = tiles < sms ? tiles : sms;
  gemm_bf16_persistent_kernel<<<grid, kThreads, smem, stream>>>(ma, mb, c, bias, M, N, K, relu, out_bf16);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { g_err = std::string("launch: ") + cudaGetErrorString(e); return -3; }
  return 0;
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

}  // namespace gemm

extern "C" {

int b2_gemm_available() { return gemm::get_encode() != nullptr; }
const char* b2_gemm_last_error() { return gemm::g_err.c_str(); }

int b2_gemm_bf16_launch(const void* a, const void* b, void* c, const float* bias, int M, int N, int K, int relu,
                        int out_bf16, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0 || (K % 8) != 0) { gemm::g_err = "bad shape (K must be a multiple of 8)"; return -4; }
  if (((uintptr_t)a | (uintptr_t)b) & 15) { gemm::g_err = "operands must be 16-byte aligned"; return -5; }
  static const int mode = [] { const char* e = getenv("B200DIST_GEMM_PERSISTENT"); return e ? atoi(e) : 1; }();
  // persistent 128x256 tiles: for at least one wave of tiles and a long K loop; small GEMMs stay on 128xBN tiles
  if (mode && N >= 192 && K >= 2048 && (long long)((M + 127) / 128) * ((N + 255) / 256) >= gemm::sm_count())
    return gemm::launch_persistent(a, b, c, bias, M, N, K, relu, out_bf16, stream);
  if (N <= 32) return gemm::launch<32>(a, b, c, bias, M, N, K, relu, out_bf16, stream);
  if (N <= 64) return gemm::launch<64>(a, b, c, bias, M, N, K, relu, out_bf16, stream);
  return gemm::launch<128>(a, b, c, bias, M, N, K, relu, out_bf16, stream);
}

}  // extern "C"
