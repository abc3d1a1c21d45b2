// Layout probes for the sm_90a tensor-core path: every assumption about TMA swizzle images and wgmma shared-memory
// descriptors is checked on hardware by tests/test_gpu_tc_probe.py, independently of the training kernels that rely on it.
//
//   tma_probe  : ONE cp.async.bulk.tensor.{2..5}d box load with a caller-defined tensor map (uint16 elements, so values are
//                exact) -> raw shared-memory image of the box, as TMA wrote it (swizzle included).
//   wgmma_probe: caller-provided shared-memory images of A and B, the A operand major and a list of
//                (A descriptor, B descriptor, accumulate) m64nNk16 MMAs of one warpgroup -> dump of D [64 x N] fp32.
//                Descriptors are given relative to the image (start address = byte offset in the image); the kernel
//                adds the shared-memory base.  Any operand major / swizzle / LBO / SBO hypothesis is testable from Python.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstring>
#include <string>

#include "tc_common.cuh"

namespace probe {

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

__global__ void __launch_bounds__(128, 1)
tma_probe_kernel(const __grid_constant__ CUtensorMap map, int rank, int c0, int c1, int c2, int c3, int c4, uint32_t bytes,
                 uint8_t* __restrict__ out) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* tile = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t bar;
  for (uint32_t i = threadIdx.x; i < bytes; i += blockDim.x) tile[i] = 0xEE;     // poison: bytes TMA did not write stay 0xEE
  if (threadIdx.x == 0) { tc::mbar_init(&bar, 1); tc::mbar_fence_init(); }
  tc::fence_proxy_async();
  __syncthreads();
  if (threadIdx.x == 0) {
    tc::mbar_expect_tx(&bar, bytes);
    const uint32_t dst = tc::smem_u32(tile), b = tc::smem_u32(&bar);
    if (rank == 2)
      asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                   ::"r"(dst), "l"(&map), "r"(b), "r"(c0), "r"(c1) : "memory");
    else if (rank == 3)
      asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                   ::"r"(dst), "l"(&map), "r"(b), "r"(c0), "r"(c1), "r"(c2) : "memory");
    else if (rank == 4)
      asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                   ::"r"(dst), "l"(&map), "r"(b), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
    else
      asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
                   ::"r"(dst), "l"(&map), "r"(b), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
  }
  tc::mbar_wait(&bar, 0);
  for (uint32_t i = threadIdx.x; i < bytes; i += blockDim.x) out[i] = tile[i];
}

struct MmaOp {
  uint64_t adesc, bdesc;     // start-address fields relative to the A / B image
  uint32_t accumulate;
};
constexpr int kMaxOps = 64;
struct MmaList {
  MmaOp op[kMaxOps];
  int n;
};

template <int N>
__global__ void __launch_bounds__(128, 1)
wgmma_probe_kernel(const uint8_t* __restrict__ a_img, uint32_t a_bytes, const uint8_t* __restrict__ b_img, uint32_t b_bytes,
                   uint32_t a_mn, const __grid_constant__ MmaList ops, float* __restrict__ dump) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sa = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sb = sa + ((a_bytes + 1023) & ~1023u);
  const int t = threadIdx.x;
  for (uint32_t i = t; i < a_bytes / 16; i += blockDim.x) reinterpret_cast<uint4*>(sa)[i] = reinterpret_cast<const uint4*>(a_img)[i];
  for (uint32_t i = t; i < b_bytes / 16; i += blockDim.x) reinterpret_cast<uint4*>(sb)[i] = reinterpret_cast<const uint4*>(b_img)[i];
  tc::fence_proxy_async();
  __syncthreads();
  const uint64_t abase = (uint64_t)((tc::smem_u32(sa) & 0x3FFFF) >> 4), bbase = (uint64_t)((tc::smem_u32(sb) & 0x3FFFF) >> 4);
  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  tc::wg_fence();
  for (int i = 0; i < ops.n; ++i)
    tc::mma<N>(d, ops.op[i].adesc + abase, ops.op[i].bdesc + bbase, ops.op[i].accumulate, a_mn);
  tc::wg_commit();
  tc::wg_wait_all();
  tc::acc_fence<N / 2>(d);
#pragma unroll
  for (int i = 0; i < N / 2; ++i) dump[tc::acc_row(t, i) * N + tc::acc_col(t, i)] = d[i];
}

}  // namespace probe

extern "C" {

const char* b2_probe_last_error() { return probe::g_err.c_str(); }

// dims/strides/box: innermost first; strides in BYTES for dims 1..rank-1 (stride of dim 0 is the element size, 2 B)
int b2_tma_probe(const void* tensor, int rank, const unsigned long long* dims, const unsigned long long* strides_bytes,
                 const unsigned int* box, int swizzle, const int* coords, unsigned int bytes, unsigned char* out,
                 cudaStream_t stream) {
  auto enc = probe::get_encode();
  if (!enc) { probe::g_err = "cuTensorMapEncodeTiled not available"; return -1; }
  if (rank < 2 || rank > 5) { probe::g_err = "rank must be 2..5"; return -2; }
  CUtensorMap map;
  cuuint64_t d[5], s[4];
  cuuint32_t b[5], e[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; e[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) s[i] = strides_bytes[i];
  const CUtensorMapSwizzle sw = swizzle == 3 ? CU_TENSOR_MAP_SWIZZLE_128B : swizzle == 2 ? CU_TENSOR_MAP_SWIZZLE_64B
                                : swizzle == 1 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = enc(&map, CU_TENSOR_MAP_DATA_TYPE_UINT16, (cuuint32_t)rank, const_cast<void*>(tensor), d, s, b, e,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { probe::g_err = "cuTensorMapEncodeTiled failed: " + std::to_string((int)r); return -3; }
  const size_t smem = bytes + 1024;
  cudaFuncSetAttribute(probe::tma_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  probe::tma_probe_kernel<<<1, 128, smem, stream>>>(map, rank, coords[0], coords[1], rank > 2 ? coords[2] : 0,
                                                     rank > 3 ? coords[3] : 0, rank > 4 ? coords[4] : 0, bytes, out);
  cudaError_t ce = cudaGetLastError();
  if (ce != cudaSuccess) { probe::g_err = std::string("launch: ") + cudaGetErrorString(ce); return -4; }
  return 0;
}

// ops: n x {adesc, bdesc, accumulate} as 3 uint64 each; dump: [64 x n] fp32
int b2_wgmma_probe(const unsigned char* a_img, unsigned int a_bytes, const unsigned char* b_img, unsigned int b_bytes,
                   int a_mn, const unsigned long long* ops, int n_ops, int n, float* dump, cudaStream_t stream) {
  if (n_ops < 1 || n_ops > probe::kMaxOps || (n != 32 && n != 64 && n != 80) || (a_bytes % 16) || (b_bytes % 16)) {
    probe::g_err = "bad probe arguments (n must be 32, 64 or 80)";
    return -1;
  }
  probe::MmaList l;
  memset(&l, 0, sizeof(l));
  l.n = n_ops;
  for (int i = 0; i < n_ops; ++i) {
    l.op[i].adesc = ops[3 * i]; l.op[i].bdesc = ops[3 * i + 1]; l.op[i].accumulate = (uint32_t)ops[3 * i + 2];
  }
  const size_t smem = ((a_bytes + 1023) & ~1023u) + ((b_bytes + 1023) & ~1023u) + 1024;
  if (smem > 200 * 1024) { probe::g_err = "images too large"; return -2; }
  auto kern = n == 32 ? probe::wgmma_probe_kernel<32> : n == 64 ? probe::wgmma_probe_kernel<64> : probe::wgmma_probe_kernel<80>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  kern<<<1, 128, smem, stream>>>(a_img, a_bytes, b_img, b_bytes, (uint32_t)(a_mn != 0), l, dump);
  cudaError_t ce = cudaGetLastError();
  if (ce != cudaSuccess) { probe::g_err = std::string("launch: ") + cudaGetErrorString(ce); return -4; }
  return 0;
}

}  // extern "C"
