// FlatEMA's update (ops/optim.py): one launch over every entry of the table described in ema.h.  Two instances:
//   host-decided   (kCounter = false): the host passes copy or lerp and launches nothing on a step it skips;
//   device-counter (kCounter = true):  for a capturable optimizer, each CTA reads the optimizer's step counter t (advanced by
//                  flat_scalars_advance after the update) and skips (t % every != 0), copies (t - every <= warmup) or lerps,
//                  so a CUDA graph that holds the step and the EMA update replays across `every` and the warmup boundary.
// Both read and write only the arrays of the table; no peer memory, no host synchronisation.
#include <cuda_runtime.h>

#include "ema.h"

namespace b2 {

constexpr int kEmaThreads = 256;
constexpr int kEmaCtasPerSm = 8;

// IEEE round-to-nearest without the flush to zero of --use_fast_math: torch's lerp keeps subnormals.
__device__ __forceinline__ float ema_sub(float a, float b) {
  float r;
  asm("sub.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float ema_fma(float a, float b, float c) {
  float r;
  asm("fma.rn.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(a), "f"(b), "f"(c));
  return r;
}

// w < 0.5: fma(w, p - e, e); otherwise fma(-(p - e), 1 - w, p), computed as fma(p - e, -(1 - w), p): the same exact product,
// so the same rounding.  -(1 - w) is a sign-bit flip, so at w = 1 it is -0 and the zero product keeps torch's sign; w - 1
// would be +0 there and turn a result of -0 into +0.
struct EmaWeight {
  float w, neg_one_minus_w;
  bool small;
};

__device__ __forceinline__ float ema_lerp(float e, float p, const EmaWeight& c) {
  const float d = ema_sub(p, e);
  return c.small ? ema_fma(c.w, d, e) : ema_fma(d, c.neg_one_minus_w, p);
}

// The entry that holds index i of the concatenated vectors (kVec) or scalars: the last entry whose first index is <= i.
// Entries with no vectors (scalars) share their first index with the next entry, so the last such entry is the one that
// holds i.
template <bool kVec>
__device__ __forceinline__ int ema_find(const EmaEntry* __restrict__ t, int n, long long i) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    const long long b = kVec ? __ldg(&t[mid].vec_begin) : __ldg(&t[mid].scalar_begin);
    if (b <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

template <bool kCounter>
__global__ void __launch_bounds__(kEmaThreads) ema_kernel(const EmaEntry* __restrict__ table, int n_entries, long long n_vec,
                                                          long long n_scalar, float w, int mode,
                                                          const long long* __restrict__ counter, long long every,
                                                          long long warmup) {
  if constexpr (kCounter) {
    __shared__ int s_mode;
    if (threadIdx.x == 0) {
      const long long t = *counter;
      s_mode = (t % every != 0) ? -1 : ((t - every <= warmup) ? EMA_COPY : EMA_LERP);
    }
    __syncthreads();
    mode = s_mode;
    if (mode < 0) return;
  }
  const bool copy = mode == EMA_COPY;
  const EmaWeight c{w, __int_as_float(__float_as_int(ema_sub(1.f, w)) ^ (int)0x80000000), w < 0.5f};
  const long long stride = (long long)gridDim.x * kEmaThreads;
  const long long first = (long long)blockIdx.x * kEmaThreads + threadIdx.x;

  // the vectors: a thread's indices ascend, so it keeps its entry until it runs past it
  long long lo = 0, hi = 0;
  float4* ev = nullptr;
  const float4* pv = nullptr;
  for (long long v = first; v < n_vec; v += stride) {
    if (v >= hi) {
      const EmaEntry* en = table + ema_find<true>(table, n_entries, v);
      lo = __ldg(&en->vec_begin);
      hi = lo + __ldg(&en->n_vec);
      const long long head = __ldg(&en->head);
      ev = reinterpret_cast<float4*>(reinterpret_cast<float*>(__ldg(reinterpret_cast<const unsigned long long*>(&en->ema))) + head);
      pv = reinterpret_cast<const float4*>(
          reinterpret_cast<const float*>(__ldg(reinterpret_cast<const unsigned long long*>(&en->live))) + head);
    }
    const long long j = v - lo;
    const float4 p = pv[j];
    float4 e = p;
    if (!copy) {
      e = ev[j];
      e.x = ema_lerp(e.x, p.x, c);
      e.y = ema_lerp(e.y, p.y, c);
      e.z = ema_lerp(e.z, p.z, c);
      e.w = ema_lerp(e.w, p.w, c);
    }
    ev[j] = e;
  }

  // the scalars: every entry's unaligned head and tail, and the entries that cannot be vectorised
  for (long long s = first; s < n_scalar; s += stride) {
    const EmaEntry* en = table + ema_find<false>(table, n_entries, s);
    const long long k = s - __ldg(&en->scalar_begin);
    const long long head = __ldg(&en->head);
    const long long i = k < head ? k : k + 4 * __ldg(&en->n_vec);
    float* ep = reinterpret_cast<float*>(__ldg(reinterpret_cast<const unsigned long long*>(&en->ema)));
    const float* pp = reinterpret_cast<const float*>(__ldg(reinterpret_cast<const unsigned long long*>(&en->live)));
    const float p = pp[i];
    ep[i] = copy ? p : ema_lerp(ep[i], p, c);
  }
}

}  // namespace b2

extern "C" {

// counter == nullptr: the host-decided instance with `mode`; otherwise the device-counter instance (mode unused).
int b2_ema_launch(const b2::EmaEntry* table, int n_entries, long long n_vec, long long n_scalar, float w, int mode,
                  const long long* counter, long long every, long long warmup, cudaStream_t stream) {
  if (table == nullptr || n_entries < 1 || n_vec < 0 || n_scalar < 0 || every < 1 || warmup < 0 ||
      (counter == nullptr && mode != b2::EMA_LERP && mode != b2::EMA_COPY))
    return (int)cudaErrorInvalidValue;
  static int sms[64] = {0};
  int dev = 0;
  cudaError_t rc = cudaGetDevice(&dev);
  if (rc != cudaSuccess) return (int)rc;
  if (dev < 0 || dev >= 64) return (int)cudaErrorInvalidDevice;
  if (sms[dev] == 0) {
    rc = cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
    if (rc != cudaSuccess) return (int)rc;
  }
  const long long work = n_vec > n_scalar ? n_vec : n_scalar;
  long long blocks = (work + b2::kEmaThreads - 1) / b2::kEmaThreads;
  const long long cap = (long long)sms[dev] * b2::kEmaCtasPerSm;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  if (counter != nullptr)
    b2::ema_kernel<true><<<(unsigned)blocks, b2::kEmaThreads, 0, stream>>>(table, n_entries, n_vec, n_scalar, w, 0, counter, every,
                                                                           warmup);
  else
    b2::ema_kernel<false><<<(unsigned)blocks, b2::kEmaThreads, 0, stream>>>(table, n_entries, n_vec, n_scalar, w, mode, nullptr,
                                                                            every, warmup);
  return (int)cudaGetLastError();
}

}  // extern "C"
