// Native batch prefetcher (C++ threads + pinned staging buffers).
//
// Stands in for the reference's `torch.utils.data.DataLoader(partition, batch_size=bsz, shuffle=True)`
// (train_dist.py:89-90), whose per-sample Python __getitem__ + PIL + ToTensor + Normalize + collate costs
// milliseconds per 128-sample batch -- far more than the whole fused training step.  Here a worker
// thread gathers the uint8 images of the next batches by index, (optionally) fuses the normalisation,
// and writes them into a ring of page-locked buffers, so the training loop only issues one async H2D
// copy per step.
#include "loader.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <random>
#include <stdexcept>

namespace b2 {

NativeLoader::NativeLoader(const uint8_t* images, const int64_t* labels, int64_t item_bytes,
                           std::vector<int64_t> index, int64_t batch, int n_buffers, bool shuffle, bool drop_last,
                           bool raw_u8, float mean, float std, uint64_t seed, bool pin)
    : images_(images), labels_(labels), item_(item_bytes), index_(std::move(index)), batch_(batch),
      nbuf_(std::max(2, n_buffers)), shuffle_(shuffle), drop_last_(drop_last), raw_(raw_u8), mean_(mean),
      inv_std_(1.f / std), seed_(seed), pinned_(pin) {
  if (batch_ <= 0) throw std::invalid_argument("batch must be positive");
  const size_t xbytes = (size_t)batch_ * item_ * (raw_ ? 1 : sizeof(float));
  const size_t ybytes = (size_t)batch_ * sizeof(int64_t);
  y_offset_ = (xbytes + 255) / 256 * 256;          // one block per slot: [x | pad | y] -> ONE H2D copy per step
  block_bytes_ = y_offset_ + ybytes;
  slots_.resize(nbuf_);
  staged_.assign(nbuf_, -1);
  {
    const char* e = getenv("B200DIST_LOADER_THREADS");
    const unsigned hc = std::thread::hardware_concurrency();
    // one thread is the default (a 128 x 784 B gather with software prefetch is short next to a step); more threads
    // compete with the thread that feeds the GPU when the host has few cores -- opt in with the variable
    (void)hc;
    nworkers_ = e ? atoi(e) : 1;
    nworkers_ = std::max(1, std::min({nworkers_, 8, nbuf_ / 2}));
  }
  for (auto& s : slots_) {
    if (pinned_) {
      if (cudaHostAlloc(&s.x, block_bytes_, cudaHostAllocDefault) != cudaSuccess) {
        cudaGetLastError();
        throw std::runtime_error("cudaHostAlloc failed");
      }
    } else {
      s.x = ::operator new(block_bytes_);
    }
    s.y = reinterpret_cast<int64_t*>(static_cast<unsigned char*>(s.x) + y_offset_);
  }
  order_ = index_;
}

NativeLoader::~NativeLoader() {
  stop();
  for (auto& s : slots_) {
    if (pinned_) cudaFreeHost(s.x);
    else ::operator delete(s.x);
  }
}

int64_t NativeLoader::num_batches() const {
  const int64_t n = (int64_t)index_.size();
  return drop_last_ ? n / batch_ : (n + batch_ - 1) / batch_;
}

void NativeLoader::start_epoch(int64_t epoch) {
  stop();
  order_ = index_;
  if (shuffle_) {
    std::mt19937_64 rng(seed_ + 0x9E3779B97F4A7C15ull * (uint64_t)(epoch + 1));
    for (size_t i = order_.size(); i > 1; --i) std::swap(order_[i - 1], order_[rng() % i]);
  }
  {
    std::lock_guard<std::mutex> lk(mu_);
    consumed_ = released_ = 0;
    std::fill(staged_.begin(), staged_.end(), (int64_t)-1);
    stopping_ = false;
  }
  for (int w = 0; w < nworkers_; ++w) workers_.emplace_back([this, w] { this->run(w); });
}

void NativeLoader::fill(Slot& s, int64_t b) {
  const int64_t n = (int64_t)order_.size();
  const int64_t lo = b * batch_, hi = std::min(n, lo + batch_);
  s.count = hi - lo;
  constexpr int64_t kAhead = 6;      // a batch is a gather of random rows: keep the DRAM misses of the next rows in flight
  for (int64_t k = lo; k < hi; ++k) {
    if (k + kAhead < hi) {
      const uint8_t* nxt = images_ + order_[k + kAhead] * item_;
      for (int64_t o = 0; o < item_; o += 64) __builtin_prefetch(nxt + o, 0, 0);
      __builtin_prefetch(labels_ + order_[k + kAhead], 0, 0);
    }
    const int64_t src = order_[k];
    const uint8_t* img = images_ + src * item_;
    if (raw_) {
      std::memcpy(static_cast<uint8_t*>(s.x) + (k - lo) * item_, img, (size_t)item_);
    } else {
      float* dst = static_cast<float*>(s.x) + (k - lo) * item_;
      const float a = inv_std_ / 255.f, c = -mean_ * inv_std_;
      for (int64_t i = 0; i < item_; ++i) dst[i] = (float)img[i] * a + c;
    }
    s.y[k - lo] = labels_[src];
  }
}

void NativeLoader::run(int worker) {
  const int64_t nb = num_batches();
  for (int64_t b = worker; b < nb; b += nworkers_) {
    {
      std::unique_lock<std::mutex> lk(mu_);
      // slot b % nbuf_ is free once the batch that used it before (b - nbuf_) has been released by the consumer
      cv_.wait(lk, [&] { return stopping_ || b - released_ < nbuf_; });
      if (stopping_) return;
    }
    fill(slots_[b % nbuf_], b);
    {
      std::lock_guard<std::mutex> lk(mu_);
      staged_[b % nbuf_] = b;
    }
    cv_.notify_all();
  }
}

// Blocks until the next batch is staged; returns its slot (or -1 at end of epoch).  The slot stays valid
// until release() has been called for it (the caller releases once its H2D copy has been enqueued+synced).
int NativeLoader::next(int64_t* count) {
  const int64_t nb = num_batches();
  std::unique_lock<std::mutex> lk(mu_);
  if (consumed_ >= nb) return -1;
  const int slot = (int)(consumed_ % nbuf_);
  cv_.wait(lk, [&] { return stopping_ || staged_[slot] == consumed_; });
  if (stopping_) return -1;
  *count = slots_[slot].count;
  ++consumed_;
  return slot;
}

int64_t NativeLoader::consumed() {
  std::lock_guard<std::mutex> lk(mu_);
  return consumed_;
}

void NativeLoader::release() {
  {
    std::lock_guard<std::mutex> lk(mu_);
    if (released_ < consumed_) ++released_;
  }
  cv_.notify_all();
}

void NativeLoader::stop() {
  {
    std::lock_guard<std::mutex> lk(mu_);
    stopping_ = true;
  }
  cv_.notify_all();
  for (auto& w : workers_) if (w.joinable()) w.join();
  workers_.clear();
}

}  // namespace b2
