// Owners of key material, host and device (DESIGN.md, "Private keys on the device", K7-K9): every handle type that keeps a
// secret on the device, and every call that stages one there, goes through these types, so a new handle type inherits the
// zero-before-free policy instead of restating it.  Plain C++ over the CUDA runtime API: the library includes it, and so
// does a CPU harness that links it against a recording stand-in for the runtime.
#pragma once
#include <cuda_runtime_api.h>

#include <algorithm>
#include <cstdint>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/bftq.h"

namespace {

// Records the text bftq_last_error returns and passes the code through (defined by the file that includes this one).
int fail(int code, const std::string& msg);

// Overwrites host memory that held key material (not elided by the optimiser).
void wipe(void* p, size_t n) {
  volatile uint8_t* v = (volatile uint8_t*)p;
  for (size_t i = 0; i < n; i++) v[i] = 0;
}

// std::allocator that wipes every block before it is freed: a vector of secret words leaves no unwiped copy behind when
// it grows or is destroyed.
template <class T> struct WipingAllocator {
  using value_type = T;
  WipingAllocator() = default;
  template <class U> WipingAllocator(const WipingAllocator<U>&) {}
  T* allocate(size_t n) { return std::allocator<T>().allocate(n); }
  void deallocate(T* p, size_t n) { wipe(p, n * sizeof(T)); std::allocator<T>().deallocate(p, n); }
  template <class U> bool operator==(const WipingAllocator<U>&) const { return true; }
  template <class U> bool operator!=(const WipingAllocator<U>&) const { return false; }
};
template <class T> using WipedVector = std::vector<T, WipingAllocator<T>>;

// Sole owner of one device allocation that holds key material (move-only).  Releasing it (reset, destruction,
// move-assignment over it) zeroes the whole block on its device, synchronises, and only then frees it.
template <class T> class DeviceSecret {
 public:
  DeviceSecret() = default;
  DeviceSecret(DeviceSecret&& o) noexcept { *this = std::move(o); }
  DeviceSecret& operator=(DeviceSecret&& o) noexcept {
    if (this != &o) {
      reset();
      std::swap(p_, o.p_); std::swap(bytes_, o.bytes_); dev_ = o.dev_;
    }
    return *this;
  }
  ~DeviceSecret() { reset(); }

  T* get() const { return p_; }
  size_t bytes() const { return bytes_; }
  explicit operator bool() const { return p_ != nullptr; }

  // The first error of the zeroing, the synchronisation and the free (each is attempted).
  cudaError_t reset() {
    if (!p_) return cudaSuccess;
    cudaSetDevice(dev_);
    cudaError_t ce = cudaMemset(p_, 0, bytes_);
    const cudaError_t cs = cudaDeviceSynchronize(), cf = cudaFree(p_);
    p_ = nullptr;
    bytes_ = 0;
    return ce != cudaSuccess ? ce : cs != cudaSuccess ? cs : cf;
  }

  // A fresh block of `bytes` on `dev`, contents undefined; whatever was held before is released first.  The caller clears
  // the sticky error of a failed allocation.
  cudaError_t alloc(int dev, size_t bytes) {
    reset();
    cudaSetDevice(dev);
    void* p = nullptr;
    const cudaError_t ce = cudaMalloc(&p, bytes);
    if (ce != cudaSuccess) return ce;
    p_ = static_cast<T*>(p); bytes_ = bytes; dev_ = dev;
    return cudaSuccess;
  }

  // A block holding `head` followed by `tail_bytes` bytes of `tail` (a registered handle's device state).  Nothing is kept
  // when an allocation or a copy fails.
  template <class H> int upload(int dev, const H& head, const void* tail, size_t tail_bytes, const char* what) {
    if (alloc(dev, sizeof(H) + tail_bytes) != cudaSuccess) {
      cudaGetLastError();
      return fail(BFTQ_ERR_NOMEM, std::string(what) + ": device allocation failed");
    }
    cudaError_t ce = cudaMemcpy(p_, &head, sizeof(H), cudaMemcpyHostToDevice);
    if (ce == cudaSuccess && tail_bytes) ce = cudaMemcpy(reinterpret_cast<uint8_t*>(p_) + sizeof(H), tail, tail_bytes, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) return BFTQ_OK;
    reset();
    return fail(BFTQ_ERR_CUDA, std::string(what) + " upload: " + cudaGetErrorString(ce));
  }

  // Replaces the block by a zeroed one of `bytes` (at least the current size) holding the current contents, and releases
  // the old one.  When the allocation, the zeroing or the copy fails, the old block stays as it was and the new one is
  // released.  An error releasing the old block is reported too; the new block is kept.
  int grow(int dev, size_t bytes, const char* what) {
    DeviceSecret fresh;
    if (fresh.alloc(dev, bytes) != cudaSuccess) {
      cudaGetLastError();
      return fail(BFTQ_ERR_NOMEM, std::string(what) + ": device allocation failed");
    }
    cudaError_t ce = cudaMemset(fresh.p_, 0, bytes);
    if (ce == cudaSuccess && p_) ce = cudaMemcpy(fresh.p_, p_, bytes_, cudaMemcpyDeviceToDevice);
    if (ce != cudaSuccess) return fail(BFTQ_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(ce));
    std::swap(*this, fresh);
    ce = fresh.reset();
    return ce == cudaSuccess ? BFTQ_OK : fail(BFTQ_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(ce));
  }

 private:
  T* p_ = nullptr;
  size_t bytes_ = 0;
  int dev_ = 0;
};

// One call's device buffer for secret inputs and intermediates: segments of one allocation, 256-byte aligned, zeroed
// before anything is uploaded and zeroed again before it is freed, on every exit path.  Copies are synchronous
// cudaMemcpy calls on the legacy default stream.  Arena is not used for these: it bounces pageable host memory through
// a staging slot's pinned mirror, and nothing scrubs that mirror.
class SecretScratch {
 public:
  // Reserves `count` elements; prepare() sets *d.
  template <class U> void seg(U** d, size_t count) {
    segs_.push_back({reinterpret_cast<void**>(d), total_});
    total_ += (count * sizeof(U) + 255) & ~(size_t)255;
  }
  // Allocates and zeroes the buffer on `dev` and resolves every segment's device pointer.
  int prepare(int dev, const char* what) {
    const int rc = buf_.grow(dev, total_, what);
    if (rc) return rc;
    for (const Seg& s : segs_) *s.d = buf_.get() + s.off;
    return BFTQ_OK;
  }
  cudaError_t put(void* d, const void* h, size_t bytes) const { return bytes ? cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice) : cudaSuccess; }
  cudaError_t get(void* h, const void* d, size_t bytes) const { return bytes ? cudaMemcpy(h, d, bytes, cudaMemcpyDeviceToHost) : cudaSuccess; }

 private:
  struct Seg { void** d; size_t off; };
  std::vector<Seg> segs_;
  size_t total_ = 0;
  DeviceSecret<uint8_t> buf_;
};

// The live handles of one type that an engine must release when it shuts down.  `mu` also serialises the calls that use
// the handles' device state.  H::detach() releases the handle's device memory and sets its engine to nullptr: a handle
// that outlives its engine keeps its host half, and destroying it then frees host memory only.
template <class H> class HandleList {
 public:
  std::mutex mu;
  void add(H* h) { std::lock_guard<std::mutex> g(mu); live_.push_back(h); }
  void remove(H* h) {
    std::lock_guard<std::mutex> g(mu);
    live_.erase(std::remove(live_.begin(), live_.end(), h), live_.end());
    h->detach();
  }
  void shutdown() {
    std::lock_guard<std::mutex> g(mu);
    for (H* h : live_) h->detach();
    live_.clear();
  }

 private:
  std::vector<H*> live_;
};

}  // namespace
