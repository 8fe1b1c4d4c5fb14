// Host build of bftkv_b200/csrc/device_secret.hpp against a recording stand-in for the CUDA runtime calls it makes.
// "Device" blocks are host memory filled with 0xA5 when allocated; every runtime call is logged, the n-th one can be made
// to fail, and a free records whether the block was all zero.  operator delete is replaced the same way for the watched
// host blocks of WipedVector.  Each sh_* entry point runs one scenario and returns the log, one call per line.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <new>
#include <string>

#include "../../bftkv_b200/csrc/device_secret.hpp"

namespace {
int fail(int code, const std::string&) { return code; }

std::string g_log;
long g_calls = 0, g_fail_at = -1;
std::map<void*, size_t> g_dev;                   // live fake device blocks
std::map<void*, size_t>& watch() {              // host blocks whose release is logged (never destroyed: delete uses it)
  static auto* m = new std::map<void*, size_t>;
  return *m;
}

bool all_zero(const void* p, size_t n) {
  const uint8_t* b = (const uint8_t*)p;
  for (size_t i = 0; i < n; i++) if (b[i]) return false;
  return true;
}
void note(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
void note(const char* fmt, ...) {
  char buf[256];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_log += buf;
  g_log += '\n';
}
bool failing(const char* op) {
  if (g_calls++ != g_fail_at) return false;
  note("FAIL %s", op);
  return true;
}
void begin(long fail_at) { g_log.clear(); g_calls = 0; g_fail_at = fail_at; }
const char* end() { return g_log.c_str(); }
void mark(const char* what) { note("-- %s", what); }
uintptr_t P(const void* p) { return (uintptr_t)p; }
}  // namespace

extern "C" {
cudaError_t cudaSetDevice(int d) {
  if (failing("setDevice")) return cudaErrorInvalidDevice;
  note("setDevice %d", d);
  return cudaSuccess;
}
cudaError_t cudaMalloc(void** p, size_t n) {
  if (failing("malloc")) return cudaErrorMemoryAllocation;
  *p = malloc(n ? n : 1);
  memset(*p, 0xA5, n);
  g_dev[*p] = n;
  note("malloc %#lx %zu", P(*p), n);
  return cudaSuccess;
}
cudaError_t cudaMemset(void* p, int v, size_t n) {
  if (failing("memset")) return cudaErrorInvalidValue;
  memset(p, v, n);
  note("memset %#lx %d %zu", P(p), v, n);
  return cudaSuccess;
}
cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind k) {
  if (failing("memcpy")) return cudaErrorInvalidValue;
  memcpy(d, s, n);
  note("memcpy %#lx %#lx %zu %s", P(d), P(s), n, k == cudaMemcpyHostToDevice ? "h2d" : k == cudaMemcpyDeviceToHost ? "d2h" : "d2d");
  return cudaSuccess;
}
cudaError_t cudaDeviceSynchronize(void) {
  if (failing("sync")) return cudaErrorLaunchFailure;
  note("sync");
  return cudaSuccess;
}
cudaError_t cudaFree(void* p) {
  if (failing("free")) return cudaErrorInvalidValue;
  auto it = g_dev.find(p);
  note("free %#lx zero=%d", P(p), it != g_dev.end() && all_zero(p, it->second));
  if (it != g_dev.end()) g_dev.erase(it);
  free(p);
  return cudaSuccess;
}
cudaError_t cudaGetLastError(void) { note("getLastError"); return cudaSuccess; }
const char* cudaGetErrorString(cudaError_t) { return "injected"; }
}  // extern "C"

void operator delete(void* p) noexcept {
  auto it = watch().find(p);
  if (it != watch().end()) {
    const bool zero = all_zero(p, it->second);
    watch().erase(it);
    note("hostfree %#lx zero=%d", P(p), zero);
  }
  free(p);
}
void operator delete(void* p, size_t) noexcept { operator delete(p); }
void* operator new(size_t n) {
  void* p = malloc(n ? n : 1);
  if (!p) throw std::bad_alloc();
  return p;
}

namespace {
struct Head { uint32_t w[5]; };
struct FakeHandle {
  void* e = nullptr;
  int detached = 0;
  DeviceSecret<Head> d;
  void detach() { detached++; d.reset(); e = nullptr; }
};
// the destroy every handle type's C entry point performs
void destroy(HandleList<FakeHandle>& list, FakeHandle* h) {
  if (h->e) list.remove(h);
  delete h;
}
const uint32_t kTail[6] = {11, 12, 13, 14, 15, 16};
}  // namespace

extern "C" {
// how: 0 reset, 1 destructor, 2 move-assignment over a live block (then the moved-from and moved-to are dropped)
const char* sh_release(int how) {
  begin(-1);
  const Head h{{1, 2, 3, 4, 5}};
  {
    DeviceSecret<Head> a, b;
    a.upload(3, h, kTail, sizeof(kTail), "a");
    b.upload(5, h, kTail, 8, "b");
    note("A %#lx B %#lx", P(a.get()), P(b.get()));
    mark("release");
    if (how == 0) a.reset();
    else if (how == 2) a = std::move(b);
    else { DeviceSecret<Head> c(std::move(a)); }
    note("after a=%#lx b=%#lx", P(a.get()), P(b.get()));
    mark("scope end");
  }
  return end();
}

// upload of head + tail with the n-th runtime call failing
const char* sh_upload(long fail_at) {
  begin(fail_at);
  const Head h{{1, 2, 3, 4, 5}};
  DeviceSecret<Head> a;
  const int rc = a.upload(2, h, kTail, sizeof(kTail), "u");
  note("rc %d held=%d bytes=%zu", rc, (bool)a, a.bytes());
  if (a) note("contents %d", memcmp(a.get(), &h, sizeof(h)) == 0 && memcmp(a.get() + 1, kTail, sizeof(kTail)) == 0);
  mark("scope end");
  a.reset();
  return end();
}

// grow(from -> to bytes) of a block holding 0, 1, 2, ... with the n-th runtime call of the growth failing
const char* sh_grow(size_t from, size_t to, long fail_at) {
  begin(-1);
  DeviceSecret<uint8_t> a;
  if (from) {
    a.grow(7, from, "g");
    for (size_t i = 0; i < from; i++) a.get()[i] = (uint8_t)(i + 1);
  }
  begin(fail_at);
  note("old %#lx %zu", P(a.get()), a.bytes());
  const int rc = a.grow(7, to, "g");
  bool kept = true, zero_tail = true;
  for (size_t i = 0; i < std::min(from, a.bytes()); i++) kept = kept && a.get()[i] == (uint8_t)(i + 1);
  for (size_t i = from; i < a.bytes(); i++) zero_tail = zero_tail && a.get()[i] == 0;
  note("rc %d now %#lx %zu kept=%d zero_tail=%d", rc, P(a.get()), a.bytes(), kept, zero_tail);
  g_fail_at = -1;
  mark("scope end");
  a.reset();
  return end();
}

// A K9-shaped call: segments of several types, prepare, uploads, kernels' writes, partial downloads, scope end; the
// n-th runtime call fails.
void scratch_call() {
  SecretScratch sc;
  uint32_t *d_a, *d_c;
  uint8_t *d_b, *d_empty, *d_out;
  uint64_t* d_d;
  sc.seg(&d_a, 100);
  sc.seg(&d_b, 1);
  sc.seg(&d_empty, 0);
  sc.seg(&d_c, 64);
  sc.seg(&d_d, 33);
  sc.seg(&d_out, 512);
  if (sc.prepare(4, "s")) { note("prepare failed"); return; }
  note("seg a %#lx 400", P(d_a));
  note("seg b %#lx 1", P(d_b));
  note("seg empty %#lx 0", P(d_empty));
  note("seg c %#lx 256", P(d_c));
  note("seg d %#lx 264", P(d_d));
  note("seg out %#lx 512", P(d_out));
  note("zeroed %d", all_zero(d_a, 400) && all_zero(d_b, 1) && all_zero(d_c, 256) && all_zero(d_d, 264) && all_zero(d_out, 512));
  std::vector<uint32_t> a(100, 7), c(64, 9);
  std::vector<uint8_t> b(1, 3), out(512, 0xEE);
  auto run = [&]() -> int {
    if (sc.put(d_a, a.data(), a.size() * 4) || sc.put(d_b, b.data(), 1) || sc.put(d_empty, nullptr, 0) || sc.put(d_c, c.data(), 200)) return 1;
    for (int i = 0; i < 512; i++) d_out[i] = (uint8_t)i;                      // the kernels' output
    if (sc.get(out.data(), d_out, 300) || sc.get(out.data(), d_empty, 0)) return 1;
    return 0;
  };
  note("run %d", run());
  int copied = 0;
  while (copied < 512 && out[copied] == (uint8_t)copied) copied++;
  note("downloaded %d untouched_after=%d", copied, out[300] == 0xEE && out[511] == 0xEE);
  mark("scope end");
}
const char* sh_scratch(long fail_at) {
  begin(fail_at);
  scratch_call();
  return end();
}

// A WipedVector of secret words grown by push_back, then destroyed: every block it frees is logged.
const char* sh_wiped_vector(void) {
  begin(-1);
  {
    WipedVector<uint32_t> v;
    for (uint32_t i = 0; i < 40; i++) {
      if (v.size() == v.capacity() && v.capacity()) { watch()[v.data()] = v.capacity() * 4; note("grow from %#lx %zu", P(v.data()), v.capacity() * 4); }
      v.push_back(0xDEADBEEF + i);
    }
    watch()[v.data()] = v.capacity() * 4;
    note("destroy %#lx %zu", P(v.data()), v.capacity() * 4);
  }
  return end();
}

// Three handles registered; one destroyed while the engine lives, the list shut down, then the other two destroyed.
const char* sh_handles(void) {
  begin(-1);
  HandleList<FakeHandle> list;
  FakeHandle* h[3];
  const Head hd{{9, 9, 9, 9, 9}};
  int engine;
  for (int i = 0; i < 3; i++) {
    h[i] = new FakeHandle;
    h[i]->e = &engine;
    h[i]->d.upload(1, hd, kTail, 4 * (i + 1), "h");
    list.add(h[i]);
    note("handle %d %#lx", i, P(h[i]->d.get()));
  }
  mark("destroy 0");
  destroy(list, h[0]);
  mark("shutdown");
  list.shutdown();
  note("detached %d %d", h[1]->detached, h[2]->detached);
  mark("destroy 1 2");
  destroy(list, h[1]);
  destroy(list, h[2]);
  mark("done");
  return end();
}
}  // extern "C"
