// Point-to-point send / recv over a symmetric mailbox for sm_90a (NVLink / NVSwitch).
//
// Replaces NCCL's send / recv under the tutorial's blocking and non-blocking point-to-point calls (tuto.md:77-120) with one
// kernel on each side.  The protocol is a bounded mailbox with per-slot sequence flags and acknowledgements, the pattern of
// NCCL's "simple" protocol:
//   * every rank's mailbox holds, per source rank, kCtas x kSlots slots of kChunk bytes;
//   * the message is cut into kChunk pieces; piece k belongs to CTA k % kCtas, and each CTA cycles through its own kSlots
//     slots.  A slot is only ever written by the same CTA index of the sender and read by the same CTA index of the
//     receiver, so each (CTA, slot) pair is a single-producer single-consumer channel;
//   * the sender stores a piece into the RECEIVER's slot (16-byte vectors over NVLink), waits at a block barrier, and thread 0
//     publishes the slot's new sequence number in the receiver's flag word with st.release.sys.  Before it refills a slot it
//     waits until the receiver's acknowledgement reached the slot's previous sequence number;
//   * the receiver waits with ld.acquire.sys until the flag reaches the expected number, copies the slot out of its OWN
//     memory (.cg loads, as the other kernels read peer-written data) into the destination, waits at a block barrier, and
//     thread 0 stores the acknowledgement into the sender's pad.
// The receiver only ever reads local memory, so a small message costs one NVLink crossing (the data, then its flag).
//
// Counters (all uint32, in the mailbox's signal pad, advanced only by these kernels, compared wrap-safe like the barrier
// epochs): flag[source][slot] (written by the sender), ack[destination][slot] (written by the receiver into the sender's
// pad), and the local-only fills[destination][slot] of the sender and consumed[source][slot] of the receiver.  A CTA's next
// slot is derived from its own counters (round robin: the number of its slots whose count equals slot 0's, mod kSlots), so
// sender and receiver pick the same slot for every piece without sharing a cursor.  Both sides must pass the same byte
// count; a mismatch leaves one side spinning until B2_SPIN_LIMIT reports it.
// The protocol is model-checked in tests/test_p2p_protocol_model.py.
#include <cstdio>
#include <mutex>
#include <set>
#include "common.cuh"

namespace b2 {
namespace p2p {

// Co-residency rule: these CTAs spin on their peer, and a GPU may run one send and one receive kernel per peer at once, so
// every CTA of all of them must be resident together: 2 x (world - 1) x kCtas <= SMs (112 of 132 on an H100 SXM at 8 GPUs;
// the one-GPU emulated ring of the tests needs 2 x 8 x 8 = 128).  Whoever changes kCtas after measuring must keep it.
constexpr int kCtas = 8;                         // G: CTAs per transfer
constexpr int kSlots = 2;                        // S: slots per CTA
constexpr size_t kChunk = 64 << 10;              // CHUNK: bytes per slot
static_assert(2 * (B2_MAX_RANKS - 1) * kCtas <= 132, "co-residency: 2 x (world - 1) x kCtas must fit the H100's 132 SMs");
static_assert((kSlots & (kSlots - 1)) == 0, "kSlots divides 2^32, so the slot cursor survives the counter wrap");
constexpr int kThreads = 512;
constexpr int kUnroll = 4;                       // 16-byte loads in flight per thread before its stores
constexpr int kPerPeer = kCtas * kSlots;         // slots per (source, destination) pair

// signal-pad word offsets of the four counter arrays, each [B2_MAX_RANKS peers][kPerPeer slots]
constexpr int kFlag = 0;
constexpr int kAck = kFlag + B2_MAX_RANKS * kPerPeer;
constexpr int kFills = kAck + B2_MAX_RANKS * kPerPeer;
constexpr int kConsumed = kFills + B2_MAX_RANKS * kPerPeer;
constexpr int kPadWords = kConsumed + B2_MAX_RANKS * kPerPeer;

// A receiver's mailbox has world - 1 source regions: source s < dst at region s, s > dst at region s - 1.
__device__ __forceinline__ uint8_t* slot_base(void* box, int src, int dst, int cta) {
  const int region = src < dst ? src : src - 1;
  return reinterpret_cast<uint8_t*>(box) + ((size_t)region * kPerPeer + (size_t)cta * kSlots) * kChunk;
}

__device__ __forceinline__ uint8_t ld_cg_u8(const uint8_t* p) {
  unsigned short v;
  asm volatile("ld.global.cg.u8 %0, [%1];" : "=h"(v) : "l"(p) : "memory");
  return (uint8_t)v;
}

// The bounded spin of the barriers: wait (thread 0) until *p reached `want` (wrap-safe), else trap with a diagnostic.
__device__ __forceinline__ void wait_reached(const uint32_t* p, uint32_t want, const char* what, int rank, int peer, int slot) {
  unsigned long long spins = 0;
  while ((int32_t)(ld_acquire_sys(p) - want) < 0) {
    if (++spins > B2_SPIN_LIMIT) {
      printf("[b200dist] p2p %s: rank %d timed out waiting for rank %d (block %d slot %d, seq %u, have %u)\n", what, rank,
             peer, (int)blockIdx.x, slot, want, ld_relaxed_sys(p));
      __trap();
    }
  }
}

// One piece, by the whole CTA: `bytes` from src to dst (both 16-byte aligned); a tail of fewer than 16 bytes byte by byte.
// Every load bypasses L1: the sender's source may have been written on another stream, the receiver's slot by a peer.
__device__ __forceinline__ void copy_piece(uint8_t* dst, const uint8_t* src, size_t bytes) {
  const size_t nv = bytes / 16;
  const uint4* s = reinterpret_cast<const uint4*>(src);
  uint4* d = reinterpret_cast<uint4*>(dst);
  for (size_t v0 = threadIdx.x; v0 < nv; v0 += (size_t)kThreads * kUnroll) {
    uint4 r[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const size_t v = v0 + (size_t)u * kThreads;
      if (v < nv) r[u] = ld_cg_v4(s + v);
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const size_t v = v0 + (size_t)u * kThreads;
      if (v < nv) st_cg_v4(d + v, r[u]);
    }
  }
  const size_t tail = nv * 16 + threadIdx.x;
  if (tail < bytes) dst[tail] = ld_cg_u8(src + tail);
}

// This CTA's slot counters, and the slot its next piece goes to (the same on both sides of a pair).
__device__ __forceinline__ int load_counters(const uint32_t* words, uint32_t (&cnt)[kSlots]) {
  int same = 0;
#pragma unroll
  for (int s = 0; s < kSlots; ++s) {
    cnt[s] = words[s];
    same += cnt[s] == cnt[0];
  }
  return same % kSlots;
}

struct P2PArgs {
  PeerPtrs box;         // mailbox data of every rank
  SignalPads sig;       // mailbox signal pad of every rank
  const void* src;      // send: the message (16-byte aligned)
  void* dst;            // recv: the destination (16-byte aligned)
  size_t nbytes;
  int rank, peer;
};

// CTA c's part of one send: its pieces (k = c, c + kCtas, ...) of the `nbytes` at `src`, through its own slots of `peer`'s
// mailbox, then its fills counters.  Shared by the single-message and the batch kernel, so both store the same words.
__device__ __forceinline__ void send_pieces(const PeerPtrs& box, const SignalPads& sig, const uint8_t* src, size_t nbytes,
                                            int rank, int peer, int c) {
  const size_t n_pieces = (nbytes + kChunk - 1) / kChunk;
  uint32_t* fills = sig.pad[rank] + kFills + peer * kPerPeer + c * kSlots;
  const uint32_t* ack = sig.pad[rank] + kAck + peer * kPerPeer + c * kSlots;
  uint32_t* flag = sig.pad[peer] + kFlag + rank * kPerPeer + c * kSlots;
  uint8_t* slots = slot_base(box.p[peer], rank, peer, c);
  uint32_t cnt[kSlots];
  int s = load_counters(fills, cnt);
  for (size_t k = c; k < n_pieces; k += kCtas) {
    uint32_t seq = 0;
#pragma unroll
    for (int q = 0; q < kSlots; ++q) seq = q == s ? cnt[q] + 1u : seq;
    if (threadIdx.x == 0) wait_reached(ack + s, seq - 1u, "send", rank, peer, s);       // the slot's last piece was read
    __syncthreads();
    const size_t off = k * kChunk;
    copy_piece(slots + (size_t)s * kChunk, src + off, nbytes - off < kChunk ? nbytes - off : kChunk);
    __syncthreads();
    if (threadIdx.x == 0) st_release_sys(flag + s, seq);
#pragma unroll
    for (int q = 0; q < kSlots; ++q) cnt[q] = q == s ? seq : cnt[q];
    s = s + 1 == kSlots ? 0 : s + 1;
  }
  if (threadIdx.x == 0) {
#pragma unroll
    for (int q = 0; q < kSlots; ++q) fills[q] = cnt[q];
  }
}

// CTA c's part of one receive from `peer` into `dst`, then its consumed counters.
__device__ __forceinline__ void recv_pieces(const PeerPtrs& box, const SignalPads& sig, uint8_t* dst, size_t nbytes,
                                            int rank, int peer, int c) {
  const size_t n_pieces = (nbytes + kChunk - 1) / kChunk;
  uint32_t* consumed = sig.pad[rank] + kConsumed + peer * kPerPeer + c * kSlots;
  const uint32_t* flag = sig.pad[rank] + kFlag + peer * kPerPeer + c * kSlots;
  uint32_t* ack = sig.pad[peer] + kAck + rank * kPerPeer + c * kSlots;
  const uint8_t* slots = slot_base(box.p[rank], peer, rank, c);
  uint32_t cnt[kSlots];
  int s = load_counters(consumed, cnt);
  for (size_t k = c; k < n_pieces; k += kCtas) {
    uint32_t seq = 0;
#pragma unroll
    for (int q = 0; q < kSlots; ++q) seq = q == s ? cnt[q] + 1u : seq;
    if (threadIdx.x == 0) wait_reached(flag + s, seq, "recv", rank, peer, s);            // the piece has landed
    __syncthreads();
    const size_t off = k * kChunk;
    copy_piece(dst + off, slots + (size_t)s * kChunk, nbytes - off < kChunk ? nbytes - off : kChunk);
    __syncthreads();
    if (threadIdx.x == 0) st_release_sys(ack + s, seq);                                    // the slot may be refilled
#pragma unroll
    for (int q = 0; q < kSlots; ++q) cnt[q] = q == s ? seq : cnt[q];
    s = s + 1 == kSlots ? 0 : s + 1;
  }
  if (threadIdx.x == 0) {
#pragma unroll
    for (int q = 0; q < kSlots; ++q) consumed[q] = cnt[q];
  }
}

__global__ void __launch_bounds__(kThreads) p2p_send_kernel(P2PArgs a) {
  send_pieces(a.box, a.sig, reinterpret_cast<const uint8_t*>(a.src), a.nbytes, a.rank, a.peer, blockIdx.x);
}

__global__ void __launch_bounds__(kThreads) p2p_recv_kernel(P2PArgs a) {
  recv_pieces(a.box, a.sig, reinterpret_cast<uint8_t*>(a.dst), a.nbytes, a.rank, a.peer, blockIdx.x);
}

// ------------------------------------------------------------------------------------------------ batch
// One launch for a list of sends and receives (torch's batch_isend_irecv).  The host groups the ops into lanes, one per
// (peer, direction) the batch uses, keeping list order inside a lane, and stores them lane after lane in the kernel
// parameters.  CTA (c, L) runs lane L's ops one after another, each as CTA c of the single-message kernel would run it
// (send_pieces / recv_pieces), and skips an op that has no piece for it (c >= its piece count), as the single launch would
// not have started CTA c.  Lanes never wait for each other inside the kernel, so a batch that lists its sends before its
// receives completes whatever the message sizes: every lane is resident at once.  Splitting a batch into several launches on
// one stream would break that (two ranks that each send more than a pair's kCtas x kSlots x kChunk before receiving would
// wait for each other for ever), so a list larger than the parameter table is refused, never split.
//
// Invariant: after a batch every counter word holds what it would hold had the ops been launched one by one in list order
// (each op moves only the counters of its own (peer, direction), and a lane applies its ops in list order).  So a batch on
// one rank matches any mix of batches and single sends / receives on its peer, and the single-message protocol model
// (tests/test_p2p_protocol_model.py) covers it; tests/test_p2p_batch_model.py checks the lane schedule itself.
constexpr int kBatchCap = 256;                   // ops per batch, in the kernel parameters (4 KB of the op table)
constexpr int kMaxLanes = 2 * (B2_MAX_RANKS - 1);

struct BatchOp {
  void* msg;            // send: the message, recv: the destination (16-byte aligned)
  size_t nbytes;
};

struct P2PBatchArgs {
  PeerPtrs box;
  SignalPads sig;
  BatchOp op[kBatchCap];                         // lane after lane, list order inside a lane
  uint16_t lane_begin[kMaxLanes + 1];            // lane L holds op[lane_begin[L] .. lane_begin[L + 1])
  int8_t lane_peer[kMaxLanes];
  int8_t lane_send[kMaxLanes];
  int rank;
};

// Co-residency as for the single kernels: a batch has at most one send and one receive lane per peer, so its grid (at most
// kCtas x 2 x (world - 1)) never exceeds what one send and one receive kernel per peer would occupy.
__global__ void __launch_bounds__(kThreads) p2p_batch_kernel(const __grid_constant__ P2PBatchArgs a) {
  const int c = blockIdx.x, lane = blockIdx.y;
  const int peer = a.lane_peer[lane];
  const bool send = a.lane_send[lane] != 0;
  for (int i = a.lane_begin[lane]; i < a.lane_begin[lane + 1]; ++i) {
    const BatchOp op = a.op[i];
    if ((size_t)c * kChunk >= op.nbytes) continue;                                        // no piece for this CTA
    __syncthreads();                                  // thread 0's counter stores of the previous op, before they are read
    if (send) send_pieces(a.box, a.sig, reinterpret_cast<const uint8_t*>(op.msg), op.nbytes, a.rank, peer, c);
    else recv_pieces(a.box, a.sig, reinterpret_cast<uint8_t*>(op.msg), op.nbytes, a.rank, peer, c);
  }
}

// With lazy module loading (CUDA_MODULE_LOADING=LAZY, which torch sets by default) a kernel is loaded at its first launch,
// and loading waits for the kernels already running on the device.  A send waiting for its receive would then wait for
// ever when the receive kernel is launched for the first time behind it (the emulated ranks of one process hit this, and
// so does any process whose first receive follows a send larger than the mailbox).  So every kernel of this file is
// loaded, once per device, before the first launch of any of them.
int load_kernels() {
  static std::mutex mu;
  static std::set<int> loaded;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return (int)e;
  std::lock_guard<std::mutex> lock(mu);
  if (loaded.count(dev)) return (int)cudaSuccess;
  cudaFuncAttributes attr;
  for (const void* f : {(const void*)p2p_send_kernel, (const void*)p2p_recv_kernel, (const void*)p2p_batch_kernel}) {
    e = cudaFuncGetAttributes(&attr, f);
    if (e != cudaSuccess) return (int)e;
  }
  loaded.insert(dev);
  return (int)cudaSuccess;
}

int launch(bool send, const PeerPtrs* box, const SignalPads* sig, const void* src, void* dst, size_t nbytes, int rank,
           int peer, int world, cudaStream_t stream) {
  if (world < 2 || world > B2_MAX_RANKS || rank < 0 || rank >= world || peer < 0 || peer >= world || peer == rank)
    return (int)cudaErrorInvalidValue;
  const void* msg = send ? src : dst;
  if (box == nullptr || sig == nullptr || msg == nullptr || (uintptr_t)msg % 16 != 0) return (int)cudaErrorInvalidValue;
  if (nbytes == 0) return (int)cudaSuccess;
  if (const int e = load_kernels()) return e;
  P2PArgs a;
  a.box = *box; a.sig = *sig; a.src = src; a.dst = dst; a.nbytes = nbytes; a.rank = rank; a.peer = peer;
  const size_t n_pieces = (nbytes + kChunk - 1) / kChunk;
  const dim3 grid((unsigned)(n_pieces < (size_t)kCtas ? n_pieces : (size_t)kCtas));
  if (send) p2p_send_kernel<<<grid, kThreads, 0, stream>>>(a);
  else p2p_recv_kernel<<<grid, kThreads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

int batch_launch(const PeerPtrs* box, const SignalPads* sig, const int* send, const int* peer, void* const* msg,
                 const size_t* nbytes, int n_ops, int rank, int world, cudaStream_t stream) {
  if (world < 2 || world > B2_MAX_RANKS || rank < 0 || rank >= world || n_ops < 0 || n_ops > kBatchCap)
    return (int)cudaErrorInvalidValue;
  if (box == nullptr || sig == nullptr) return (int)cudaErrorInvalidValue;
  if (n_ops > 0 && (send == nullptr || peer == nullptr || msg == nullptr || nbytes == nullptr))
    return (int)cudaErrorInvalidValue;
  // ops with bytes per (direction, peer); the lanes are the (direction, peer) that have any: sends first, in peer order
  int count_of[2][B2_MAX_RANKS] = {};
  size_t max_pieces = 0;
  for (int i = 0; i < n_ops; ++i) {
    if ((send[i] != 0 && send[i] != 1) || peer[i] < 0 || peer[i] >= world || peer[i] == rank) return (int)cudaErrorInvalidValue;
    if (msg[i] == nullptr || (uintptr_t)msg[i] % 16 != 0) return (int)cudaErrorInvalidValue;
    if (nbytes[i] == 0) continue;
    ++count_of[send[i]][peer[i]];
    const size_t pieces = (nbytes[i] + kChunk - 1) / kChunk;
    max_pieces = pieces > max_pieces ? pieces : max_pieces;
  }
  if (max_pieces == 0) return (int)cudaSuccess;                                          // only zero-byte ops
  if (const int e = load_kernels()) return e;
  P2PBatchArgs a;
  int lane_of[2][B2_MAX_RANKS], count[kMaxLanes], n_lanes = 0;
  for (int d = 1; d >= 0; --d)
    for (int p = 0; p < world; ++p)
      if (count_of[d][p] > 0) {
        a.lane_peer[n_lanes] = (int8_t)p;
        a.lane_send[n_lanes] = (int8_t)d;
        count[n_lanes] = count_of[d][p];
        lane_of[d][p] = n_lanes++;
      }
  a.lane_begin[0] = 0;
  for (int L = 0; L < n_lanes; ++L) a.lane_begin[L + 1] = (uint16_t)(a.lane_begin[L] + count[L]);
  int fill[kMaxLanes];
  for (int L = 0; L < n_lanes; ++L) fill[L] = a.lane_begin[L];
  for (int i = 0; i < n_ops; ++i)                                                          // stable: list order per lane
    if (nbytes[i] > 0) a.op[fill[lane_of[send[i]][peer[i]]]++] = BatchOp{msg[i], nbytes[i]};
  a.box = *box; a.sig = *sig; a.rank = rank;
  // CTAs past the largest op's piece count would skip every op, as the single launches would not start them
  const dim3 grid((unsigned)(max_pieces < (size_t)kCtas ? max_pieces : (size_t)kCtas), (unsigned)n_lanes);
  p2p_batch_kernel<<<grid, kThreads, 0, stream>>>(a);
  return (int)cudaGetLastError();
}

}  // namespace p2p
}  // namespace b2

// ============================================================================================ launchers
extern "C" {

// The mailbox geometry parallel/symm.py allocates: CTAs per transfer, slots per CTA, bytes per slot, signal-pad words.
void b2_p2p_config(int* ctas, int* slots, size_t* chunk, int* pad_words) {
  *ctas = b2::p2p::kCtas;
  *slots = b2::p2p::kSlots;
  *chunk = b2::p2p::kChunk;
  *pad_words = b2::p2p::kPadWords;
}

// Send `nbytes` from `src` to rank `peer` (send), or receive them from `peer` into `dst` (recv), through the mailboxes `box`
// with signal pads `sig` (one per rank).  Both sides must pass the same byte count.  Returns cudaError_t as int; nothing is
// launched for zero bytes, and cudaErrorInvalidValue, without a launch, for a world outside 2..8, a rank or peer outside
// [0, world), peer == rank, or a missing or not 16-byte aligned message pointer.
int b2_p2p_send_launch(const PeerPtrs* box, const b2::SignalPads* sig, const void* src, size_t nbytes, int rank, int peer,
                       int world, cudaStream_t stream) {
  return b2::p2p::launch(true, box, sig, src, nullptr, nbytes, rank, peer, world, stream);
}

int b2_p2p_recv_launch(const PeerPtrs* box, const b2::SignalPads* sig, void* dst, size_t nbytes, int rank, int peer,
                       int world, cudaStream_t stream) {
  return b2::p2p::launch(false, box, sig, nullptr, dst, nbytes, rank, peer, world, stream);
}

// The most ops one b2_p2p_batch_launch takes.
int b2_p2p_batch_capacity() { return b2::p2p::kBatchCap; }

// Every op of a list in one launch: op i sends nbytes[i] from msg[i] to rank peer[i] (send[i] == 1) or receives them from
// it into msg[i] (send[i] == 0), with the counters each (peer, direction) would have after the ops one by one in list order.
// Returns cudaError_t as int; cudaErrorInvalidValue, without a launch, for a world outside 2..8, a rank or peer outside
// [0, world), peer == rank, a direction other than 0 / 1, a missing or not 16-byte aligned message pointer, or more than
// b2_p2p_batch_capacity() ops.  Zero-byte ops are no-ops, and a batch of only those launches nothing.
int b2_p2p_batch_launch(const PeerPtrs* box, const b2::SignalPads* sig, const int* send, const int* peer, void* const* msg,
                        const size_t* nbytes, int n_ops, int rank, int world, cudaStream_t stream) {
  return b2::p2p::batch_launch(box, sig, send, peer, msg, nbytes, n_ops, rank, world, stream);
}

}  // extern "C"
