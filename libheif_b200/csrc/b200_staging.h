// b200_staging.h -- host-side resources of the decoder and the host colour entry points: a persistent thread pool, owning
// handles of device buffers, streams, events and page-locked blocks, and the page-locked bounce buffer that pageable host
// memory moves through on its way to or from the device.
#pragma once
#include "b200_internal.h"
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <utility>
#include <vector>

namespace b200 {

// minimal persistent thread pool: parallel_for over [0, n)
class Pool {
 public:
  explicit Pool(int n) : stop_(false), gen_(0), next_(0), total_(0), pending_(0) { for (int i = 0; i < n; i++) th_.emplace_back([this] { run(); }); }
  ~Pool() { { std::lock_guard<std::mutex> l(mu_); stop_ = true; } cv_.notify_all(); for (auto& t : th_) t.join(); }
  int size() const { return (int)th_.size(); }
  void parallel_for(int n, const std::function<void(int)>& fn) {
    if (n <= 0) return;
    if (th_.empty() || n == 1) { for (int i = 0; i < n; i++) fn(i); return; }
    { std::lock_guard<std::mutex> l(mu_); fn_ = &fn; total_ = n; next_.store(0); pending_ = (int)th_.size(); gen_++; }
    cv_.notify_all();
    std::unique_lock<std::mutex> l(mu_);
    done_.wait(l, [this] { return pending_ == 0; });
  }
 private:
  void run() {
    unsigned seen = 0;
    for (;;) {
      const std::function<void(int)>* fn; int total;
      { std::unique_lock<std::mutex> l(mu_); cv_.wait(l, [&] { return stop_ || gen_ != seen; }); if (stop_) return; seen = gen_; fn = fn_; total = total_; }
      for (;;) { int i = next_.fetch_add(1); if (i >= total) break; (*fn)(i); }
      { std::lock_guard<std::mutex> l(mu_); if (--pending_ == 0) done_.notify_all(); }
    }
  }
  std::vector<std::thread> th_; std::mutex mu_; std::condition_variable cv_, done_;
  bool stop_; unsigned gen_; std::atomic<int> next_; int total_, pending_; const std::function<void(int)>* fn_ = nullptr;
};

template <typename T>
struct DevBuf {   // grow-only device buffer with optional pinned host staging of the same capacity; owns both (move-only)
  T* d = nullptr; T* h = nullptr; size_t cap = 0, hcap = 0;
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : d(o.d), h(o.h), cap(o.cap), hcap(o.hcap) { o.d = o.h = nullptr; o.cap = o.hcap = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept { std::swap(d, o.d); std::swap(h, o.h); std::swap(cap, o.cap); std::swap(hcap, o.hcap); return *this; }
  ~DevBuf() { if (d) cudaFree(d); if (h) cudaFreeHost(h); }
  int reserve(size_t n, bool host = true) {
    if (n > cap) {
      const size_t nc = n + n / 4 + 1024;
      if (d) cudaFree(d);
      d = nullptr; cap = 0;
      B200_CUDA_CHECK(cudaMalloc(&d, nc * sizeof(T)));
      cap = nc;
    }
    if (host && n > hcap) {
      if (h) cudaFreeHost(h);
      h = nullptr; hcap = 0;
      B200_CUDA_CHECK(cudaMallocHost(&h, cap * sizeof(T)));
      hcap = cap;
    }
    return B200_OK;
  }
};

// owning handle of a stream, an event or a page-locked block
template <typename H, cudaError_t (*Destroy)(H)>
struct Owned {
  H h = nullptr;
  Owned() = default;
  Owned(const Owned&) = delete;
  Owned& operator=(const Owned&) = delete;
  ~Owned() { if (h) Destroy(h); }
  operator H() const { return h; }
};
template <typename T>
cudaError_t free_pinned(T* p) { return cudaFreeHost(p); }
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
using Event = Owned<cudaEvent_t, cudaEventDestroy>;
template <typename T>
using Pinned = Owned<T*, free_pinned<T>>;

// Whether the device can copy to / from `p` directly: page-locked (cudaHostAlloc, cudaHostRegister) or managed memory.
bool is_page_locked(const void* p);

// Moves 2-D host regions to / from the device.  Page-locked or managed operands are copied directly (queued on the stream).
// Pageable ones go through two page-locked slots in bands of rows: the pool's threads copy band k while the DMA engine moves
// band k - 1.  A slot holds 32 MiB, or one row if a row is longer.  upload() returns once the last band is queued,
// download() once every band is in place.  All calls on one Bounce must use the same stream: download() relies on stream
// order to reuse a slot an upload is still reading.
class Bounce {
 public:
  int upload(void* dst, size_t dpitch, const void* src, size_t sstride, size_t wb, size_t h, cudaStream_t s, Pool& pool);
  int download(void* dst, size_t dstride, const void* src, size_t spitch, size_t wb, size_t h, cudaStream_t s, Pool& pool);
 private:
  int reserve(size_t wb);       // slots of at least one row of wb bytes
  uint8_t* slot(unsigned k) const { return pin_.h + (size_t)k * slot_bytes_; }
  Pinned<uint8_t> pin_;
  size_t slot_bytes_ = 0;
  Event ev_[2];                 // the last copy into / out of each slot
  bool ev_used_[2] = {false, false};
  unsigned next_ = 0;           // upload: the slot the next band goes into
};

}  // namespace b200
