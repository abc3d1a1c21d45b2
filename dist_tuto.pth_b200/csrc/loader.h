// Native batch prefetcher -- see loader.cpp.
#pragma once
#include <condition_variable>
#include <cstdint>
#include <mutex>
#include <thread>
#include <vector>

namespace b2 {

class NativeLoader {
 public:
  struct Slot {
    void* x = nullptr;       // [batch, item] float32 (normalised) or uint8 (raw)
    int64_t* y = nullptr;    // [batch]
    int64_t count = 0;
  };
  NativeLoader(const uint8_t* images, const int64_t* labels, int64_t item_bytes, std::vector<int64_t> index,
               int64_t batch, int n_buffers, bool shuffle, bool drop_last, bool raw_u8, float mean, float std,
               uint64_t seed, bool pin);
  ~NativeLoader();
  int64_t num_batches() const;
  void start_epoch(int64_t epoch);
  int next(int64_t* count);
  int64_t consumed();            // batches handed out this epoch (slot of batch b = b % num_slots())
  void release();
  void stop();
  const Slot& slot(int i) const { return slots_[i]; }
  int num_slots() const { return nbuf_; }
  size_t y_offset() const { return y_offset_; }
  size_t block_bytes() const { return block_bytes_; }
  int64_t batch() const { return batch_; }
  int64_t item() const { return item_; }
  bool raw() const { return raw_; }
  bool pinned() const { return pinned_; }

 private:
  void run(int worker);
  void fill(Slot& s, int64_t b);
  const uint8_t* images_;
  const int64_t* labels_;
  int64_t item_;
  std::vector<int64_t> index_, order_;
  int64_t batch_;
  int nbuf_;
  bool shuffle_, drop_last_, raw_;
  float mean_, inv_std_;
  uint64_t seed_;
  bool pinned_;
  size_t y_offset_ = 0, block_bytes_ = 0;
  std::vector<Slot> slots_;
  // `nworkers_` prefetch threads: worker w stages batches w, w + nworkers_, ... (a random-index gather of 128 x 784 B is
  // DRAM-latency bound on one core: ~30 us per batch, i.e. slower than the GPU step); batches are handed out in order.
  int nworkers_ = 1;
  std::vector<std::thread> workers_;
  std::vector<int64_t> staged_;      // per slot: index of the batch currently staged in it (-1: none)
  std::mutex mu_;
  std::condition_variable cv_;
  int64_t consumed_ = 0, released_ = 0;
  bool stopping_ = true;
};

}  // namespace b2
