// b200_staging.cc -- the page-locked bounce buffer of b200_staging.h
#include "b200_staging.h"
#include <algorithm>

namespace b200 {

namespace {
constexpr size_t kSlotBytes = (size_t)32 << 20;
constexpr size_t kParallelBytes = (size_t)1 << 20;     // smaller bands are copied on the calling thread

// rows of wb bytes, split over the pool's threads
void copy_rows(Pool& pool, uint8_t* dst, size_t dstride, const uint8_t* src, size_t sstride, size_t wb, size_t rows) {
  const size_t parts = rows * wb < kParallelBytes ? 1 : std::max<size_t>(1, std::min<size_t>(rows, (size_t)pool.size()));
  pool.parallel_for((int)parts, [&](int t) {
    for (size_t r = rows * (size_t)t / parts, r1 = rows * (size_t)(t + 1) / parts; r < r1; r++) memcpy(dst + r * dstride, src + r * sstride, wb);
  });
}
}  // namespace

bool is_page_locked(const void* p) {
  cudaPointerAttributes pa{};
  const bool pinned = cudaPointerGetAttributes(&pa, p) == cudaSuccess && (pa.type == cudaMemoryTypeHost || pa.type == cudaMemoryTypeManaged);
  cudaGetLastError();
  return pinned;
}

int Bounce::reserve(size_t wb) {
  if (!ev_[0].h)
    for (Event& e : ev_) B200_CUDA_CHECK(cudaEventCreateWithFlags(&e.h, cudaEventDisableTiming));
  const size_t need = std::max(kSlotBytes, wb);
  if (need <= slot_bytes_) return B200_OK;
  for (int k = 0; k < 2; k++)                          // no copy may still use the old slots
    if (ev_used_[k]) B200_CUDA_CHECK(cudaEventSynchronize(ev_[k]));
  if (pin_.h) cudaFreeHost(pin_.h);
  pin_.h = nullptr; slot_bytes_ = 0;
  B200_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&pin_.h), 2 * need, cudaHostAllocDefault));
  slot_bytes_ = need;
  return B200_OK;
}

int Bounce::upload(void* dst, size_t dpitch, const void* src, size_t sstride, size_t wb, size_t h, cudaStream_t s, Pool& pool) {
  if (!wb || !h) return B200_OK;
  if (is_page_locked(src)) { B200_CUDA_CHECK(cudaMemcpy2DAsync(dst, dpitch, src, sstride, wb, h, cudaMemcpyHostToDevice, s)); return B200_OK; }
  int rc;
  if ((rc = reserve(wb))) return rc;
  const size_t band = slot_bytes_ / wb;
  for (size_t y0 = 0; y0 < h; y0 += band) {
    const unsigned k = next_++ & 1u;
    const size_t n = std::min(band, h - y0);
    if (ev_used_[k]) B200_CUDA_CHECK(cudaEventSynchronize(ev_[k]));      // the copy that last used this slot is done
    copy_rows(pool, slot(k), wb, static_cast<const uint8_t*>(src) + y0 * sstride, sstride, wb, n);
    B200_CUDA_CHECK(cudaMemcpy2DAsync(static_cast<uint8_t*>(dst) + y0 * dpitch, dpitch, slot(k), wb, wb, n, cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaEventRecord(ev_[k], s));
    ev_used_[k] = true;
  }
  return B200_OK;
}

int Bounce::download(void* dst, size_t dstride, const void* src, size_t spitch, size_t wb, size_t h, cudaStream_t s, Pool& pool) {
  if (!wb || !h) return B200_OK;
  if (is_page_locked(dst)) { B200_CUDA_CHECK(cudaMemcpy2DAsync(dst, dstride, src, spitch, wb, h, cudaMemcpyDeviceToHost, s)); return B200_OK; }
  int rc;
  if ((rc = reserve(wb))) return rc;
  const size_t band = slot_bytes_ / wb, nb = (h + band - 1) / band;
  for (size_t k = 0; k <= nb; k++) {
    if (k < nb) {                                      // queue band k into slot k & 1 (band k - 2, its previous content, was drained in iteration k - 1)
      const size_t y0 = k * band;
      B200_CUDA_CHECK(cudaMemcpy2DAsync(slot(k & 1), wb, static_cast<const uint8_t*>(src) + y0 * spitch, spitch, wb, std::min(band, h - y0), cudaMemcpyDeviceToHost, s));
      B200_CUDA_CHECK(cudaEventRecord(ev_[k & 1], s));
      ev_used_[k & 1] = true;
    }
    if (k > 0) {                                       // band k - 1 has arrived: drain it while band k is in flight
      const size_t j = k - 1, y0 = j * band;
      B200_CUDA_CHECK(cudaEventSynchronize(ev_[j & 1]));
      copy_rows(pool, static_cast<uint8_t*>(dst) + y0 * dstride, dstride, slot(j & 1), wb, wb, std::min(band, h - y0));
    }
  }
  return B200_OK;
}

}  // namespace b200
