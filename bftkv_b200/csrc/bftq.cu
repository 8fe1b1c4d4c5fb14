// libbftq.so — C ABI (include/bftq.h) over the sm_90a kernels.
// Host side: engine life cycle, key table (per-key Montgomery constants), launch plumbing,
// pinned staging.  No CPU verification path exists here on purpose.
#include "../../include/bftq.h"
#include "rsa_verify.cuh"
#include "rsa_verify_r32.cuh"
#include "tally.cuh"
#include "lagrange.cuh"
#include "modexp.cuh"
#include "ed25519_fast.cuh"
#include "p256.cuh"
#include "dsa_verify.cuh"
#include "pgp_digest.cuh"
#include "pgp_parse.cuh"
#include "msg_parse.cuh"
#include "msg_decrypt.cuh"
#include "thrsa_sign.cuh"
#include "thdsa_sign.cuh"
#include "auth_server.cuh"
#include "auth_client.cuh"
#include "data_encrypt.cuh"
#include "pgp_host.hpp"
#include "wotqs_host.hpp"
#include "bignum_host.hpp"
#include "device_secret.hpp"
#include "wire_host.hpp"
#include "thdsa_wire.hpp"

#include <algorithm>
#include <array>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <set>
#include <thread>
#include <mutex>
#include <string>
#include <vector>

#include <sched.h>
#include <unistd.h>

namespace {

thread_local std::string g_last_error;

int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}
#define CU(call)                                                                              \
  do {                                                                                        \
    cudaError_t _e = (call);                                                                  \
    if (_e != cudaSuccess)                                                                    \
      return fail(BFTQ_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e));         \
  } while (0)

// Tunables from the environment (INTEGRATION.md lists them).  Each caller decides WHEN its variable is read: a function
// static reads it once per process, a plain call on every use.
bool env_set(const char* name) { return getenv(name) != nullptr; }
// A positive number, else the default.
uint64_t env_u64(const char* name, uint64_t dflt) {
  const char* v = getenv(name);
  const long long x = v ? atoll(v) : 0;
  return x > 0 ? (uint64_t)x : dflt;
}
// A switch that is on by default stays on unless set to 0; one that is off by default stays off unless set to a positive number.
bool env_on(const char* name, bool dflt) {
  const char* v = getenv(name);
  if (!v) return dflt;
  return dflt ? atoi(v) != 0 : atoi(v) > 0;
}

using namespace bftq::hostbig;

void to_digits(const UBig& a, uint32_t* d, int nd) {
  for (int i = 0; i < nd; i++) {
    int o = 28 * i;
    uint32_t v = 0;
    if (o < 64 * kHL) {
      int wi = o >> 6, sh = o & 63;
      unsigned __int128 t = a.w[wi];
      if (wi + 1 < kHL) t |= (unsigned __int128)a.w[wi + 1] << 64;
      v = (uint32_t)(t >> sh) & bftq::kDigitMask;
    }
    d[i] = v;
  }
}

struct StagingSlot {
  cudaStream_t stream = nullptr;
  uint8_t* h_pinned = nullptr;  size_t h_cap = 0;
  uint8_t* d_buf = nullptr;     size_t d_cap = 0;
  cudaEvent_t done = nullptr;   // blocking-sync event: a waiting packer thread sleeps instead of spinning
  bool busy = false;
};

}  // namespace

// Persistent host workers for the packet-level entry points.  A batch call posts a job (its worker body) and
// works on it itself; idle pool threads join the oldest job that still has chunks to hand out.  Threads are
// created once (spawning them per call costs a noticeable share of a batch) and keep their per-thread caches.
struct PackerPool {
  struct Job {
    std::function<void()> body;
    std::function<bool()> has_work;          // false once every chunk has been handed out
    unsigned max_joiners = 0, joined = 0;    // pool threads allowed to / that did join (under PackerPool::mu)
    unsigned active = 0;                     // pool threads currently inside body()
  };
  std::mutex mu;
  std::condition_variable cv_jobs, cv_idle;
  std::deque<std::shared_ptr<Job>> jobs;
  std::vector<std::thread> threads;
  bool stop = false;
  std::function<void()> on_start;            // run once by every pool thread (NUMA binding to the engine's GPU)

  void ensure(unsigned n) {                  // grow to n threads (under mu)
    while (threads.size() < n) threads.emplace_back([this] { loop(); });
  }
  void loop() {
    if (on_start) on_start();
    std::unique_lock<std::mutex> l(mu);
    for (;;) {
      std::shared_ptr<Job> j;
      cv_jobs.wait(l, [&] {
        if (stop) return true;
        for (auto& c : jobs) if (c->joined < c->max_joiners && c->has_work()) { j = c; return true; }
        return false;
      });
      if (stop) return;
      j->joined++; j->active++;
      l.unlock();
      j->body();
      l.lock();
      j->active--;
      cv_idle.notify_all();
    }
  }
  // Runs body on the calling thread and on up to `helpers` pool threads; returns when all of them are out.
  void run(unsigned helpers, std::function<void()> body, std::function<bool()> has_work) {
    auto j = std::make_shared<Job>();
    j->body = body; j->has_work = std::move(has_work); j->max_joiners = helpers;
    if (helpers) {
      std::lock_guard<std::mutex> l(mu);
      ensure(helpers);
      jobs.push_back(j);
    }
    if (helpers) cv_jobs.notify_all();
    body();
    if (!helpers) return;
    std::unique_lock<std::mutex> l(mu);
    for (auto it = jobs.begin(); it != jobs.end(); ++it) if (*it == j) { jobs.erase(it); break; }
    cv_idle.wait(l, [&] { return j->active == 0; });
  }
  ~PackerPool() {
    { std::lock_guard<std::mutex> l(mu); stop = true; }
    cv_jobs.notify_all();
    for (auto& t : threads) t.join();
  }
};

// Ed25519 window-table cache (see ed_cache_prepare).
struct EdCache {
  std::mutex mu;
  bftq::ed::gea* d_tab = nullptr;                // cap_slots x FxA::entries entries of 128 bytes (keys)
  bftq::ed::gea* d_tabB = nullptr;               // FxB::entries entries (the base point)
  bftq::EdSlotHdr* d_hdr = nullptr;
  uint32_t cap_slots = 0, used = 0;
  uint64_t builds = 0;                           // tables built so far
  uint64_t resets = 0;                           // times a full cache was emptied for a batch that pays for its tables
  std::map<std::string, uint32_t> slot_of;       // 32 key bytes -> slot
  std::vector<cudaEvent_t> pending;              // builds that may still be running
  bool enabled = true;                           // BFTQ_ED25519_TABLES, read when the engine is created
};

// Large device scratch blocks kept across calls (bftq_read_responses_batch needs about 2.5 x the raw answers; a
// cudaMalloc / cudaFree pair of a gigabyte per call costs milliseconds and serialises on the driver's allocator lock).
struct ScratchCache {
  std::mutex mu;
  std::vector<std::pair<void*, size_t>> free_list;     // at most kKeep blocks
  static constexpr size_t kKeep = 3;
};

// The bftq_stats counters.  Relaxed atomics: worker threads count without taking a lock, and no reader needs one counter
// ordered against another.
struct EngineStats {
  struct Counter {
    std::atomic<uint64_t> v{0};
    void operator+=(uint64_t x) { v.fetch_add(x, std::memory_order_relaxed); }
    operator uint64_t() const { return v.load(std::memory_order_relaxed); }
  };
  Counter items, launches, h2d_bytes, d2h_bytes, packer_chunks, packer_parse_ns, packer_stage_ns, packer_wait_ns,
      msg_gpu_items, msg_host_items, unsupported_items;
};

// mu guards the published key table (keys, key_lookup, n_dev_keys, all_2048, retired), the staging slots, the DSA key
// table, the certificate-constant cache and host_allocs.  Counters and verify flags are atomics and take no lock.
struct bftq_engine {
  int device = 0;
  EdCache ed;
  ScratchCache scratch;
  int sm_count = 0;
  std::mutex mu;
  std::vector<bftq::RsaKeyDev> h_keys;
  bftq::RsaKeyDev* d_keys = nullptr;
  size_t d_keys_cap = 0;
  std::vector<bftq::r32::RsaKey32> h_keys32;     // radix-2^32 constants of the same keys
  bftq::r32::RsaKey32* d_keys32 = nullptr;
  std::vector<void*> retired;                    // device key tables replaced by larger ones (freed at shutdown)
  size_t n_dev_keys = 0;                         // keys fully uploaded and published (what a launch may index)
  bool all_2048 = true;                          // every registered modulus has exactly 2048 bits
  // Montgomery constants of keys that arrive with a call (VerifyWithCertificate's presented certificate): a bounded
  // host-side cache, never entered in the device table above (an unauthenticated presenter must not grow engine state)
  std::map<std::string, std::pair<bftq::RsaKeyDev, bftq::r32::RsaKey32>> cert_consts;
  std::vector<StagingSlot*> slots;
  EngineStats stats;
  std::map<std::string, uint32_t> key_lookup;   // (modulus bytes || e) -> key table index
  struct DsaKey { std::vector<uint8_t> p, q, gy; int cls; };   // gy: g || y, each padded to |p| bytes
  std::vector<DsaKey> dsa_keys;                  // host table; a group's domain travels with its launch
  std::map<std::string, uint32_t> dsa_lookup;
  PackerPool pool;                               // host workers of the packet-level entry points
  // NUMA placement: the CPUs of the node the GPU hangs off (intersected with the process's affinity mask).  The pool's
  // threads are bound to them and pinned staging memory is allocated from a thread bound to them, so that staging
  // copies and the DMA engine read node-local memory (8-GPU boxes: GPUs 4-7 sit on the second socket).
  int numa_node = -1;
  bool numa_valid = false;
  cpu_set_t numa_cpus;
  std::map<void*, size_t> host_allocs;           // bftq_host_alloc blocks
  std::atomic<uint32_t> packer_flags{0};   // BFTQ_F_* the packet-level entry points pass to K1 (bftq_engine_set_verify_flags / env BFTQ_STRICT_RANGE)
  // live handles that hold key material on the device, zeroed and freed at shutdown
  HandleList<bftq_keyring> keyrings;             // private-key tables
  HandleList<bftq_thrsa_share> thrsa;            // threshold-RSA fragments
  HandleList<bftq_thdsa_share> thdsa;            // threshold-DSA Y and (k, c) tables; mu also covers the sign calls
  HandleList<bftq_auth_server> auth;             // auth parameters and phase-1 state; mu also covers the respond calls
  HandleList<bftq_auth_client> auth_client;      // auth client sessions; mu also covers the process calls
  uint32_t* d_p256_base = nullptr;               // K8's fixed-base table of P-256 (public), built on first use
  bftq::k9::AuthGroup* d_auth_group = nullptr;   // K9's group constants (public), built on first use
  bftq::k9::AuthGroup* d_auth_group_q = nullptr; // K10's constants of q = (p - 1) / 2 (public), built on first use
};

namespace {

// Blocks for n items at one item per thread.
unsigned grid_per_item(uint64_t n, int block) { return (unsigned)((n + block - 1) / block); }
// Blocks for n items at per_block items per block, at most per_sm blocks per SM and at least one: the kernel strides over
// the rest.
unsigned grid_capped(const bftq_engine* e, uint64_t n, uint64_t per_block, uint64_t per_sm) {
  return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((n + per_block - 1) / per_block, (uint64_t)std::max(1, e->sm_count) * per_sm));
}
// Every kernel the library launches goes through here (bftq_measure_int_peak's timed loop aside): the launch is checked,
// and counted in bftq_stats' launches.
template <typename... P, typename... A>
int launch(bftq_engine* e, const char* name, void (*kernel)(P...), unsigned blocks, unsigned threads, cudaStream_t st, A&&... args) {
  kernel<<<blocks, threads, 0, st>>>(std::forward<A>(args)...);
  const cudaError_t ce = cudaGetLastError();
  if (ce != cudaSuccess) return fail(BFTQ_ERR_CUDA, std::string(name) + " launch: " + cudaGetErrorString(ce));
  e->stats.launches += 1;
  return BFTQ_OK;
}
// One of the engine's lazily built public tables (freed at shutdown); nothing stays allocated when the upload fails.
template <class T> int upload_table(const T* host, size_t count, T** out, const char* what) {
  T* d = nullptr;
  if (cudaMalloc(&d, count * sizeof(T)) != cudaSuccess) { cudaGetLastError(); return fail(BFTQ_ERR_NOMEM, std::string(what) + ": device allocation failed"); }
  if (cudaMemcpy(d, host, count * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(d); return fail(BFTQ_ERR_CUDA, std::string(what) + " upload failed"); }
  *out = d;
  return BFTQ_OK;
}

// A device block of at least `bytes` (the smallest cached one that fits, else a fresh cudaMalloc).  The caller must have
// finished every stream that touched the block before releasing it.
void* scratch_acquire(bftq_engine* e, size_t bytes, size_t* got) {
  {
    std::lock_guard<std::mutex> g(e->scratch.mu);
    int best = -1;
    for (int i = 0; i < (int)e->scratch.free_list.size(); i++)
      if (e->scratch.free_list[i].second >= bytes && (best < 0 || e->scratch.free_list[i].second < e->scratch.free_list[best].second)) best = i;
    if (best >= 0) {
      const auto b = e->scratch.free_list[best];
      e->scratch.free_list.erase(e->scratch.free_list.begin() + best);
      *got = b.second;
      return b.first;
    }
  }
  void* p = nullptr;
  const size_t want = bytes + bytes / 8;                 // headroom: the next batch is rarely byte-identical in size
  if (cudaMalloc(&p, want) == cudaSuccess) { *got = want; return p; }
  cudaGetLastError();
  {                                                      // out of memory: drop the cache and ask for the exact size
    std::lock_guard<std::mutex> g(e->scratch.mu);
    for (auto& b : e->scratch.free_list) cudaFree(b.first);
    e->scratch.free_list.clear();
  }
  if (cudaMalloc(&p, bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  *got = bytes;
  return p;
}
void scratch_release(bftq_engine* e, void* p, size_t bytes) {
  if (!p) return;
  void* drop = nullptr;
  {
    std::lock_guard<std::mutex> g(e->scratch.mu);
    e->scratch.free_list.emplace_back(p, bytes);
    if (e->scratch.free_list.size() > ScratchCache::kKeep) {
      int small = 0;
      for (int i = 1; i < (int)e->scratch.free_list.size(); i++) if (e->scratch.free_list[i].second < e->scratch.free_list[small].second) small = i;
      drop = e->scratch.free_list[small].first;
      e->scratch.free_list.erase(e->scratch.free_list.begin() + small);
    }
  }
  if (drop) cudaFree(drop);
}

void numa_probe(bftq_engine* e) {
  e->numa_valid = false;
  if (!env_on("BFTQ_NUMA_BIND", true)) return;
  char bdf[32] = {0};
  if (cudaDeviceGetPCIBusId(bdf, sizeof(bdf), e->device) != cudaSuccess) { cudaGetLastError(); return; }
  for (char* c = bdf; *c; c++) *c = (char)tolower(*c);
  char path[128];
  snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bdf);
  int node = -1;
  if (FILE* f = fopen(path, "r")) { if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f); }
  e->numa_node = node;
  if (node < 0) return;
  snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
  FILE* f = fopen(path, "r");
  if (!f) return;
  char list[4096] = {0};
  const size_t got = fread(list, 1, sizeof(list) - 1, f);
  fclose(f);
  list[got] = 0;
  cpu_set_t node_cpus, mine;
  CPU_ZERO(&node_cpus);
  for (char* tok = strtok(list, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
    int a = 0, b = 0;
    const int k = sscanf(tok, "%d-%d", &a, &b);
    if (k == 1) b = a;
    if (k >= 1) for (int c = a; c <= b && c < CPU_SETSIZE; c++) CPU_SET(c, &node_cpus);
  }
  if (sched_getaffinity(0, sizeof(mine), &mine) != 0) return;
  CPU_AND(&e->numa_cpus, &node_cpus, &mine);
  e->numa_valid = CPU_COUNT(&e->numa_cpus) > 0 && CPU_COUNT(&e->numa_cpus) < CPU_COUNT(&mine);   // nothing to gain when the mask is the node already
}
void numa_bind_this_thread(bftq_engine* e) {
  if (e && e->numa_valid) sched_setaffinity(0, sizeof(e->numa_cpus), &e->numa_cpus);
}
// Runs the enclosing scope on the GPU's NUMA node (page-locked allocations land where the allocating thread runs).
struct ScopedNumaBind {
  cpu_set_t saved; bool active = false;
  explicit ScopedNumaBind(bftq_engine* e) {
    if (e && e->numa_valid && sched_getaffinity(0, sizeof(saved), &saved) == 0) { active = sched_setaffinity(0, sizeof(e->numa_cpus), &e->numa_cpus) == 0; }
  }
  ~ScopedNumaBind() { if (active) sched_setaffinity(0, sizeof(saved), &saved); }
};

// Picks a free staging slot: the smallest one that is already large enough, else the largest free one
// (which then grows), else a new one.  Growing means cudaFreeHost / cudaHostAlloc / cudaMalloc — calls that
// stall the whole device — so capacities are rounded up to a power of two (at least 1 MiB): calls of varying
// size settle on a stable pool after a few batches instead of reallocating for ever.
int acquire_slot(bftq_engine* e, size_t h_bytes, size_t d_bytes, StagingSlot** out) {
  StagingSlot* s = nullptr;
  {
    std::lock_guard<std::mutex> g(e->mu);
    StagingSlot *fit = nullptr, *big = nullptr;
    for (auto* c : e->slots) {
      if (c->busy) continue;
      if (c->h_cap >= h_bytes && c->d_cap >= d_bytes) { if (!fit || c->h_cap < fit->h_cap) fit = c; }
      else if (!big || c->h_cap > big->h_cap) big = c;
    }
    s = fit ? fit : big;
    if (!s) { s = new StagingSlot(); e->slots.push_back(s); }
    s->busy = true;
  }
  auto round_up = [](size_t v) { size_t c = (size_t)1 << 20; while (c < v) c <<= 1; return c; };
  CU(cudaSetDevice(e->device));
  if (!s->stream) CU(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
  if (!s->done) CU(cudaEventCreateWithFlags(&s->done, cudaEventBlockingSync | cudaEventDisableTiming));
  if (s->h_cap < h_bytes) {
    if (s->h_pinned) cudaFreeHost(s->h_pinned);
    s->h_pinned = nullptr; s->h_cap = 0;
    const size_t cap = round_up(h_bytes);
    ScopedNumaBind on_node(e);
    CU(cudaHostAlloc((void**)&s->h_pinned, cap, cudaHostAllocDefault));
    s->h_cap = cap;
  }
  if (s->d_cap < d_bytes) {
    if (s->d_buf) cudaFree(s->d_buf);
    s->d_buf = nullptr; s->d_cap = 0;
    const size_t cap = round_up(d_bytes);
    CU(cudaMalloc((void**)&s->d_buf, cap));
    s->d_cap = cap;
  }
  *out = s;
  return BFTQ_OK;
}

// A call's staging plan: device buffers carved out of one slot, inputs uploaded in one go,
// outputs downloaded in one go.  Pinned caller memory is DMA'd directly, pageable memory is
// bounced through the slot's pinned mirror.
class Arena {
 public:
  explicit Arena(bftq_engine* e) : e_(e) {}
  // Work may have been enqueued without finish() having run (an error path returned early): nothing may reuse, regrow
  // or free the slot's buffers — or the caller's output bounce — under kernels and copies still in flight.
  ~Arena() {
    if (!s_) return;
    if (enqueued_ && s_->stream) cudaStreamSynchronize(s_->stream);
    std::lock_guard<std::mutex> g(e_->mu);
    s_->busy = false;
  }
  // count = elements reserved on the device, copy = elements actually copied (defaults to count)
  template <typename T> void in(T** dptr, const T* host, size_t count, size_t copy = (size_t)-1) {
    add((void**)dptr, (void*)host, count * sizeof(T), (copy == (size_t)-1 ? count : copy) * sizeof(T), true);
  }
  template <typename T> void out(T** dptr, T* host, size_t count, size_t copy = (size_t)-1) {
    add((void**)dptr, (void*)host, count * sizeof(T), (copy == (size_t)-1 ? count : copy) * sizeof(T), false);
  }
  // An input the caller composes in place: after prepare(), *hptr is the slot's pinned mirror of the
  // buffer (write `count` elements there), so the bytes cross host memory once.
  template <typename T> void stage(T** dptr, T** hptr, size_t count) {
    add((void**)dptr, nullptr, count * sizeof(T), count * sizeof(T), true);
    bufs_.back().hptr = (void**)hptr;
  }
  cudaStream_t stream() const { return s_->stream; }
  // Acquires the staging slot and resolves every device (and staged host) pointer.  upload() calls it
  // when the caller has not.
  int prepare() {
    if (s_) return BFTQ_OK;
    int rc = acquire_slot(e_, total_, total_, &s_);
    if (rc) return rc;
    for (auto& b : bufs_) {
      *b.dptr = s_->d_buf + b.off;
      if (b.hptr) { *b.hptr = s_->h_pinned + b.off; b.host = s_->h_pinned + b.off; }
    }
    return BFTQ_OK;
  }
  int upload() {
    int rc = prepare();
    if (rc) return rc;
    enqueued_ = true;
    uint64_t h2d = 0;
    // Inputs that live in the slot's pinned mirror (staged in place or bounced) have the same layout on
    // both sides, so neighbours travel in ONE copy: a chunk of the packer costs one H2D call, not nine
    // (driver calls from many worker threads serialise on the context lock).
    size_t run_lo = (size_t)-1, run_hi = 0;
    auto flush = [&]() -> cudaError_t {
      if (run_lo == (size_t)-1) return cudaSuccess;
      cudaError_t ce = cudaMemcpyAsync(s_->d_buf + run_lo, s_->h_pinned + run_lo, run_hi - run_lo, cudaMemcpyHostToDevice, s_->stream);
      run_lo = (size_t)-1;
      return ce;
    };
    for (auto& b : bufs_) {
      if (!b.is_in || b.copy == 0) continue;
      h2d += b.copy;
      if (!b.hptr && is_pinned(b.host)) {                      // caller's pinned memory: DMA straight from it
        CU(cudaMemcpyAsync(s_->d_buf + b.off, b.host, b.copy, cudaMemcpyHostToDevice, s_->stream));
        continue;
      }
      if (!b.hptr) memcpy(s_->h_pinned + b.off, b.host, b.copy);
      if (run_lo != (size_t)-1 && b.off - run_hi > 65536) CU(flush());      // do not drag a large output region along
      if (run_lo == (size_t)-1) run_lo = b.off;
      run_hi = b.off + b.copy;
    }
    CU(flush());
    e_->stats.h2d_bytes += h2d;
    return BFTQ_OK;
  }
  int download() {
    int rc = download_async();
    if (rc) return rc;
    return finish();
  }
  // enqueue the device-to-host copies without waiting (finish() waits and un-bounces)
  int download_async() {
    uint64_t d2h = 0;
    bounce_.clear();
    for (auto& b : bufs_) {
      if (b.is_in || b.copy == 0) continue;
      if (is_pinned(b.host)) {
        CU(cudaMemcpyAsync(b.host, s_->d_buf + b.off, b.copy, cudaMemcpyDeviceToHost, s_->stream));
      } else {
        CU(cudaMemcpyAsync(s_->h_pinned + b.off, s_->d_buf + b.off, b.copy, cudaMemcpyDeviceToHost, s_->stream));
        bounce_.push_back(&b);
      }
      d2h += b.copy;
    }
    if (sleepy_) { CU(cudaEventRecord(s_->done, s_->stream)); recorded_ = true; }
    e_->stats.d2h_bytes += d2h;
    return BFTQ_OK;
  }
  // sleepy = wait on a blocking-sync event (the thread sleeps until the copy has landed) instead of spinning
  // in cudaStreamSynchronize: the packer's workers share the host's CPU quota with the threads still parsing.
  void set_sleepy(bool v) { sleepy_ = v; }
  int finish() {
    if (!s_) return BFTQ_OK;                          // nothing was enqueued (prepare() failed or was never called)
    if (sleepy_ && recorded_) CU(cudaEventSynchronize(s_->done));
    else CU(cudaStreamSynchronize(s_->stream));
    enqueued_ = false;
    for (auto* b : bounce_) memcpy(b->host, s_->h_pinned + b->off, b->copy);
    bounce_.clear();
    return BFTQ_OK;
  }

 private:
  struct Buf { void** dptr; void* host; size_t off, bytes, copy; bool is_in; void** hptr; };
  void add(void** dptr, void* host, size_t bytes, size_t copy, bool is_in) {
    bufs_.push_back({dptr, host, total_, bytes, copy, is_in, nullptr});
    total_ += (bytes + 255) & ~(size_t)255;
  }
  static bool is_pinned(const void* p) {
    cudaPointerAttributes at;
    const bool pinned = cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type == cudaMemoryTypeHost;
    cudaGetLastError();
    return pinned;
  }
  bftq_engine* e_;
  StagingSlot* s_ = nullptr;
  bool sleepy_ = false, recorded_ = false, enqueued_ = false;
  std::vector<Buf> bufs_;
  std::vector<const Buf*> bounce_;
  size_t total_ = 0;
};

// A host batch travels as chunks through a ring of four staging slots, one stream each: the copies of chunk c + 1 run
// under the kernels of chunk c, and kernels of neighbouring chunks run out of phase.
struct ArenaRing {
  bftq_engine* e;
  std::unique_ptr<Arena> slots[4];
  uint64_t n = 0;
  Arena& next(int& rc) {                       // the oldest chunk is finished (rc: its result) and a fresh arena takes its place
    std::unique_ptr<Arena>& slot = slots[n++ % 4];
    rc = slot ? slot->finish() : (int)BFTQ_OK;
    slot.reset(new Arena(e));
    return *slot;
  }
  int drain(int rc) {                          // finishes every chunk still in flight; the first error (rc included) wins
    for (auto& slot : slots) if (slot) { const int r2 = slot->finish(); if (!rc) rc = r2; slot.reset(); }
    return rc;
  }
};
// Items per chunk of such a batch (tools/e2e_experiment.py compares one unchunked call with four 16384-item pieces in
// flight); BFTQ_HOST_CHUNK overrides, read once per process.
uint64_t host_chunk() { static const uint64_t n = env_u64("BFTQ_HOST_CHUNK", 16384); return n; }

// The key table a launch indexes: a consistent snapshot of the engine's published table (taken under e->mu), or the
// table of one call (keys presented with the call).
struct KeyView {
  const bftq::RsaKeyDev* d_keys = nullptr;
  const bftq::r32::RsaKey32* d_keys32 = nullptr;
  uint32_t nkeys = 0;
  bool all_2048 = true;
};
KeyView global_keys(bftq_engine* e) {
  std::lock_guard<std::mutex> g(e->mu);
  return KeyView{e->d_keys, e->d_keys32, (uint32_t)e->n_dev_keys, e->all_2048};
}

template <int T, int W, int BLOCK, int KB>
int launch_rsa(bftq_engine* e, const KeyView& kv, const uint32_t* d_key_idx, const uint8_t* d_sig, const uint8_t* d_digest,
               uint32_t hash_alg, uint64_t n_items, uint32_t flags, const uint8_t* d_pre, uint8_t* d_status, cudaStream_t st) {
  auto kern = bftq::rsa_verify_kernel<T, W, BLOCK, KB>;
  static thread_local int occ = 0;
  if (!occ) { CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, BLOCK, 0)); if (occ < 1) occ = 1; }
  return launch(e, "rsa_verify_kernel", kern, grid_capped(e, n_items, (BLOCK / 32) * (32 / T), occ), BLOCK, st, kv.d_keys, kv.nkeys,
                d_key_idx, d_sig, d_digest, hash_alg, n_items, flags, d_pre, d_status);
}

// exact2048: -1 = decide from the table (every key has exactly 2048 bits), 1 = the caller knows that every key this
// launch touches has (the packer groups by key), 0 = some do not (radix-2^28 kernel).
int launch_rsa_any(bftq_engine* e, const KeyView& kv, const uint32_t* d_key_idx, const uint8_t* d_sig, const uint8_t* d_digest,
                   uint32_t hash_alg, uint64_t n_items, uint32_t flags, const uint8_t* d_pre, uint8_t* d_status, cudaStream_t st,
                   int kb = 256, int exact2048 = -1) {
  if (!kv.d_keys || !kv.d_keys32) return fail(BFTQ_ERR_INVALID_ARG, "no keys registered");
  e->stats.items += n_items;
  const bool fits32 = exact2048 < 0 ? kv.all_2048 : exact2048 == 1;
  if (kb == 256 && fits32) {
    constexpr int blk = bftq::r32::kK1Block;
    static thread_local int occ32 = 0;
    if (!occ32) { CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ32, bftq::r32::rsa_verify_r32_kernel, blk, 0)); if (occ32 < 1) occ32 = 1; }
    return launch(e, "rsa_verify_r32_kernel", bftq::r32::rsa_verify_r32_kernel, grid_capped(e, n_items, (blk / 32) * 8, occ32), blk, st,
                  kv.d_keys32, kv.nkeys, d_key_idx, d_sig, d_digest, hash_alg, n_items, flags, d_pre, d_status);
  }
  switch (kb) {
    case 128: return launch_rsa<4, 10, 128, 128>(e, kv, d_key_idx, d_sig, d_digest, hash_alg, n_items, flags, d_pre, d_status, st);
    case 192: return launch_rsa<4, 14, 128, 192>(e, kv, d_key_idx, d_sig, d_digest, hash_alg, n_items, flags, d_pre, d_status, st);
    case 256: return launch_rsa<4, 19, 128, 256>(e, kv, d_key_idx, d_sig, d_digest, hash_alg, n_items, flags, d_pre, d_status, st);
    case 384: return launch_rsa<8, 14, 128, 384>(e, kv, d_key_idx, d_sig, d_digest, hash_alg, n_items, flags, d_pre, d_status, st);
    case 512: return launch_rsa<8, 19, 128, 512>(e, kv, d_key_idx, d_sig, d_digest, hash_alg, n_items, flags, d_pre, d_status, st);
    default: return fail(BFTQ_ERR_UNSUPPORTED_KEY, "key size class not built (128/192/256/384/512 bytes are)");
  }
}

// ---- integer-pipe peak micro-benchmark ---------------------------------------------------------
// The roofline denominator: the rate of the instruction K1's products are made of, IMAD.WIDE.U32.X (a
// mad.lo.cc/madc.hi.cc pair).  Two independent carry chains x, y of four pairs per thread, eight steps per
// loop trip, all inside ONE asm block with its own registers: with the accumulators in C variables ptxas
// renames them through IMAD.MOV on the same pipe and the kernel under-reads the peak.  The loop must hold
// the 64 wide multiplies and nothing else on that pipe (tests/test_abi.py checks the SASS).
#define BFTQ_PEAK_PAIR(op, lo, hi, a) op " " lo ", " a ", %4, " lo ";\n\tmadc.hi.cc.u32 " hi ", " a ", %4, " hi ";\n\t"
#define BFTQ_PEAK_CHAIN(r)                                                                                         \
  BFTQ_PEAK_PAIR("mad.lo.cc.u32", r "0", r "1", "%1") BFTQ_PEAK_PAIR("madc.lo.cc.u32", r "2", r "3", "%2")         \
  BFTQ_PEAK_PAIR("madc.lo.cc.u32", r "4", r "5", "%3") BFTQ_PEAK_PAIR("madc.lo.cc.u32", r "6", r "7", "%5")        \
  "addc.u32 " r "8, " r "8, 0;\n\t"
#define BFTQ_PEAK_STEP BFTQ_PEAK_CHAIN("x") BFTQ_PEAK_CHAIN("y")
constexpr int kPeakMacsPerIter = 8;     // one BFTQ_PEAK_STEP
constexpr int kPeakUnroll = 8;          // steps per loop trip; iters must be a multiple

__global__ void __launch_bounds__(256) int_peak_kernel(uint32_t* out, uint32_t seed, int iters) {
  const uint32_t x = seed * 2654435761u + threadIdx.x;
  uint32_t s;
  asm volatile(
      "{\n\t.reg .u32 x0, x1, x2, x3, x4, x5, x6, x7, x8, y0, y1, y2, y3, y4, y5, y6, y7, y8;\n\t.reg .u32 n;\n\t.reg .pred p;\n\t"
      "add.u32 x0, %7, 1;\n\t" "add.u32 y0, %7, 101;\n\t"
      "add.u32 x1, %7, 2;\n\t" "add.u32 y1, %7, 102;\n\t"
      "add.u32 x2, %7, 3;\n\t" "add.u32 y2, %7, 103;\n\t"
      "add.u32 x3, %7, 4;\n\t" "add.u32 y3, %7, 104;\n\t"
      "add.u32 x4, %7, 5;\n\t" "add.u32 y4, %7, 105;\n\t"
      "add.u32 x5, %7, 6;\n\t" "add.u32 y5, %7, 106;\n\t"
      "add.u32 x6, %7, 7;\n\t" "add.u32 y6, %7, 107;\n\t"
      "add.u32 x7, %7, 8;\n\t" "add.u32 y7, %7, 108;\n\t"
      "add.u32 x8, %7, 9;\n\t" "add.u32 y8, %7, 109;\n\t"
      "mov.u32 n, %6;\n"
      "PEAK_LOOP_%=:\n\t"
      BFTQ_PEAK_STEP BFTQ_PEAK_STEP BFTQ_PEAK_STEP BFTQ_PEAK_STEP BFTQ_PEAK_STEP BFTQ_PEAK_STEP BFTQ_PEAK_STEP BFTQ_PEAK_STEP
      "sub.u32 n, n, 8;\n\t"
      "setp.gt.s32 p, n, 0;\n\t"
      "@p bra PEAK_LOOP_%=;\n\t"
      "xor.b32 %0, x0, y0;\n\t" "xor.b32 %0, %0, x1;\n\t" "xor.b32 %0, %0, y1;\n\t" "xor.b32 %0, %0, x2;\n\t"
      "xor.b32 %0, %0, y2;\n\t" "xor.b32 %0, %0, x3;\n\t" "xor.b32 %0, %0, y3;\n\t" "xor.b32 %0, %0, x4;\n\t"
      "xor.b32 %0, %0, y4;\n\t" "xor.b32 %0, %0, x5;\n\t" "xor.b32 %0, %0, y5;\n\t" "xor.b32 %0, %0, x6;\n\t"
      "xor.b32 %0, %0, y6;\n\t" "xor.b32 %0, %0, x7;\n\t" "xor.b32 %0, %0, y7;\n\t" "xor.b32 %0, %0, x8;\n\t"
      "xor.b32 %0, %0, y8;\n\t}"
      : "=r"(s)
      : "r"(x ^ 0x243f6a88u), "r"(x ^ 0x85a308d3u), "r"(x ^ 0x13198a2eu), "r"(x | 1u), "r"(x ^ 0x03707344u), "r"(iters), "r"(x));
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
#undef BFTQ_PEAK_STEP
#undef BFTQ_PEAK_CHAIN
#undef BFTQ_PEAK_PAIR

}  // namespace

extern "C" {

int bftq_version(void) { return BFTQ_VERSION; }
const char* bftq_last_error(void) { return g_last_error.c_str(); }

int bftq_init(int device, bftq_engine** out) {
  if (!out) return fail(BFTQ_ERR_INVALID_ARG, "out is NULL");
  *out = nullptr;
  int count = 0;
  cudaError_t ce = cudaGetDeviceCount(&count);
  if (ce != cudaSuccess || count == 0)
    return fail(BFTQ_ERR_NO_DEVICE, std::string("no CUDA device: ") + cudaGetErrorString(ce));
  if (device < 0 || device >= count) return fail(BFTQ_ERR_INVALID_ARG, "device ordinal out of range");
  CU(cudaSetDevice(device));
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)      // the library carries sm_90a code only, which loads on no other architecture
    return fail(BFTQ_ERR_NO_DEVICE, std::string("device is not sm_90 (Hopper): ") + prop.name);
  auto* e = new bftq_engine();
  e->device = device;
  e->sm_count = prop.multiProcessorCount;
  if (env_on("BFTQ_STRICT_RANGE", false)) e->packer_flags |= BFTQ_F_STRICT_RANGE;
  e->ed.enabled = env_on("BFTQ_ED25519_TABLES", true);
  numa_probe(e);
  e->pool.on_start = [e] { numa_bind_this_thread(e); };
  *out = e;
  return BFTQ_OK;
}

int bftq_host_alloc(bftq_engine* e, uint64_t bytes, void** out) {
  if (!e || !out) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  *out = nullptr;
  CU(cudaSetDevice(e->device));
  void* p = nullptr;
  {
    ScopedNumaBind on_node(e);
    CU(cudaHostAlloc(&p, (size_t)std::max<uint64_t>(bytes, 1), cudaHostAllocPortable));
  }
  std::lock_guard<std::mutex> g(e->mu);
  e->host_allocs[p] = (size_t)bytes;
  *out = p;
  return BFTQ_OK;
}
int bftq_host_free(bftq_engine* e, void* p) {
  if (!e) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (!p) return BFTQ_OK;
  {
    std::lock_guard<std::mutex> g(e->mu);
    auto it = e->host_allocs.find(p);
    if (it == e->host_allocs.end()) return fail(BFTQ_ERR_INVALID_ARG, "not a bftq_host_alloc block of this engine");
    e->host_allocs.erase(it);
  }
  CU(cudaSetDevice(e->device));
  CU(cudaFreeHost(p));
  return BFTQ_OK;
}
int bftq_bind_thread(bftq_engine* e) {
  if (!e) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  numa_bind_this_thread(e);
  return e->numa_valid ? e->numa_node : -1;
}

int bftq_device_sm_count(bftq_engine* e) { return e ? e->sm_count : BFTQ_ERR_INVALID_ARG; }
int bftq_engine_set_verify_flags(bftq_engine* e, uint32_t flags) {
  if (!e || (flags & ~(uint32_t)BFTQ_F_STRICT_RANGE)) return fail(BFTQ_ERR_INVALID_ARG, "unknown flag");
  e->packer_flags = flags;
  return BFTQ_OK;
}
int bftq_key_count(bftq_engine* e) {
  if (!e) return BFTQ_ERR_INVALID_ARG;
  std::lock_guard<std::mutex> g(e->mu);
  return (int)e->n_dev_keys;
}

int bftq_register_rsa_keys(bftq_engine* e, const uint8_t* n_be, const uint32_t* exps, uint32_t count,
                           uint32_t* first_index) {
  return bftq_register_rsa_keys_k(e, n_be, 256, exps, count, first_index);
}

}  // extern "C"
namespace {
// Per-key Montgomery constants for both kernel families from a big-endian modulus.  *is2048: exactly 2048 bits.
int make_key_consts(const uint8_t* n_be, uint32_t stride, uint32_t exp, bftq::RsaKeyDev& kd, bftq::r32::RsaKey32& k32, bool* is2048) {
  UBig n;
  from_be(n, n_be, stride);
  const int nb = bitlen(n);
  const int kb = (nb + 7) / 8;
  const int cls = bftq::class_of(kb);
  if (!cls || !(n.w[0] & 1)) return fail(BFTQ_ERR_UNSUPPORTED_KEY, "modulus must be odd and at most 4096 bits");
  if (exp == 0) return fail(BFTQ_ERR_UNSUPPORTED_KEY, "public exponent 0");
  memset(&kd, 0, sizeof(kd));
  to_digits(n, kd.n, bftq::kMaxDigits);
  const uint32_t n0inv = neg_inv32((uint32_t)n.w[0]);
  kd.n0inv = n0inv & bftq::kDigitMask;                   // -n^-1 mod 2^28 for the digit kernels
  kd.e = exp;
  kd.nbits = (uint32_t)nb;
  kd.kbytes = (uint32_t)kb;
  // R^2 mod n for the class's digit layout: 2^(2*28*digits) by repeated doubling from 1.
  UBig one;
  memset(&one, 0, sizeof(one));
  one.w[0] = 1;
  to_digits(shl_mod(one, n, 2 * 28 * bftq::class_digits(cls)), kd.r2, bftq::kMaxDigits);
  // radix-2^32 constants (fast path, meaningful for exactly-2048-bit moduli): n, -n^-1 mod 2^32, the verification constants
  memset(&k32, 0, sizeof(k32));
  to_words(n, k32.n, 64);
  k32.n0inv = n0inv;
  k32.e = exp;
  k32.nbits = (uint32_t)nb;
  if (nb == 2048) {
    const bftq::hostbig::VerifyConsts vc = bftq::hostbig::verify_consts(n, exp);
    to_words(vc.c16, k32.c16, 64);
    to_words(vc.hc16, k32.hc16, 64);
    to_words(vc.c32, k32.c32, 64);
    to_words(vc.hc32, k32.hc32, 64);
  }
  if (is2048) *is2048 = !(cls == 256 && nb != 2048);
  return BFTQ_OK;
}
}  // namespace
extern "C" {

int bftq_register_rsa_keys_k(bftq_engine* e, const uint8_t* n_be, uint32_t stride, const uint32_t* exps, uint32_t count,
                             uint32_t* first_index) {
  if (!e || !n_be || !exps) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (stride == 0 || stride > 512) return fail(BFTQ_ERR_INVALID_ARG, "modulus stride must be 1..512 bytes");
  std::vector<bftq::RsaKeyDev> fresh(count);
  std::vector<bftq::r32::RsaKey32> fresh32(count);
  bool fresh_all_2048 = true;
  for (uint32_t k = 0; k < count; k++) {
    bool is2048 = true;
    const int rc = make_key_consts(n_be + (size_t)k * stride, stride, exps[k], fresh[k], fresh32[k], &is2048);
    if (rc) return fail(rc, g_last_error + " (key " + std::to_string(k) + ")");
    fresh_all_2048 = fresh_all_2048 && is2048;
  }
  // Publication order (launchers snapshot {pointers, count, all_2048} under the same mutex, global_keys()): the new
  // keys are on the device — synchronously — BEFORE the count that makes them reachable moves, a larger table is
  // complete before its pointer replaces the old one, and host state changes only after every CUDA call succeeded.
  std::lock_guard<std::mutex> g(e->mu);
  CU(cudaSetDevice(e->device));
  const size_t old = e->n_dev_keys, want = old + count;
  if (want > e->d_keys_cap) {
    // Kernels in flight may still read the old table: it is retired, not freed (released at bftq_shutdown).  The
    // table grows only with the keyring (keys that arrive with a call never enter it), so this is bounded.
    const size_t cap = std::max<size_t>(64, want * 2);
    bftq::RsaKeyDev* nd = nullptr;
    bftq::r32::RsaKey32* nd32 = nullptr;
    if (cudaMalloc((void**)&nd, cap * sizeof(bftq::RsaKeyDev)) != cudaSuccess) return fail(BFTQ_ERR_NOMEM, "key table allocation failed");
    if (cudaMalloc((void**)&nd32, cap * sizeof(bftq::r32::RsaKey32)) != cudaSuccess) { cudaFree(nd); return fail(BFTQ_ERR_NOMEM, "key table allocation failed"); }
    cudaError_t ce = cudaSuccess;
    if (old) {
      ce = cudaMemcpy(nd, e->h_keys.data(), old * sizeof(bftq::RsaKeyDev), cudaMemcpyHostToDevice);
      if (ce == cudaSuccess) ce = cudaMemcpy(nd32, e->h_keys32.data(), old * sizeof(bftq::r32::RsaKey32), cudaMemcpyHostToDevice);
    }
    if (ce == cudaSuccess && count) ce = cudaMemcpy(nd + old, fresh.data(), count * sizeof(bftq::RsaKeyDev), cudaMemcpyHostToDevice);
    if (ce == cudaSuccess && count) ce = cudaMemcpy(nd32 + old, fresh32.data(), count * sizeof(bftq::r32::RsaKey32), cudaMemcpyHostToDevice);
    if (ce != cudaSuccess) { cudaFree(nd); cudaFree(nd32); return fail(BFTQ_ERR_CUDA, std::string("key table upload: ") + cudaGetErrorString(ce)); }
    if (e->d_keys) e->retired.push_back(e->d_keys);
    if (e->d_keys32) e->retired.push_back(e->d_keys32);
    e->d_keys = nd;
    e->d_keys32 = nd32;
    e->d_keys_cap = cap;
  } else if (count) {
    // slots [old, want) are beyond every published count: no launch reads them yet
    CU(cudaMemcpy(e->d_keys + old, fresh.data(), count * sizeof(bftq::RsaKeyDev), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(e->d_keys32 + old, fresh32.data(), count * sizeof(bftq::r32::RsaKey32), cudaMemcpyHostToDevice));
  }
  e->h_keys.insert(e->h_keys.end(), fresh.begin(), fresh.end());
  e->h_keys32.insert(e->h_keys32.end(), fresh32.begin(), fresh32.end());
  e->all_2048 = e->all_2048 && fresh_all_2048;
  e->n_dev_keys = want;
  if (first_index) *first_index = (uint32_t)old;
  return BFTQ_OK;
}

int bftq_rsa_verify_batch_dev(bftq_engine* e, const uint32_t* d_key_idx, const uint8_t* d_sig_be,
                              const uint8_t* d_digest, uint32_t hash_alg, uint64_t n_items, uint32_t flags,
                              uint8_t* d_status, void* cuda_stream) {
  return bftq_rsa_verify_batch_dev_k(e, 256, d_key_idx, d_sig_be, d_digest, hash_alg, n_items, flags, d_status, cuda_stream);
}

int bftq_rsa_verify_batch_dev_k(bftq_engine* e, uint32_t key_bytes, const uint32_t* d_key_idx, const uint8_t* d_sig_be,
                                const uint8_t* d_digest, uint32_t hash_alg, uint64_t n_items, uint32_t flags,
                                uint8_t* d_status, void* cuda_stream) {
  if (!bftq::class_supported((int)key_bytes)) return fail(BFTQ_ERR_UNSUPPORTED_KEY, "key size class not built");
  if (!e || !d_key_idx || !d_sig_be || !d_digest || !d_status) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (bftq::host_hash_dlen(hash_alg) == 0) return fail(BFTQ_ERR_INVALID_ARG, "unknown hash algorithm id");
  if (n_items == 0) return BFTQ_OK;
  CU(cudaSetDevice(e->device));
  return launch_rsa_any(e, global_keys(e), d_key_idx, d_sig_be, d_digest, hash_alg, n_items, flags, nullptr, d_status, (cudaStream_t)cuda_stream, (int)key_bytes);
}

int bftq_rsa_verify_batch(bftq_engine* e, const uint32_t* key_idx, const uint8_t* sig_be, const uint8_t* digest,
                          uint32_t hash_alg, uint64_t n_items, uint32_t flags, uint8_t* out_status) {
  return bftq_rsa_verify_batch_k(e, 256, key_idx, sig_be, digest, hash_alg, n_items, flags, out_status);
}

int bftq_rsa_verify_batch_k(bftq_engine* e, uint32_t key_bytes, const uint32_t* key_idx, const uint8_t* sig_be, const uint8_t* digest,
                            uint32_t hash_alg, uint64_t n_items, uint32_t flags, uint8_t* out_status) {
  if (!e || !key_idx || !sig_be || !digest || !out_status) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (!bftq::class_supported((int)key_bytes)) return fail(BFTQ_ERR_UNSUPPORTED_KEY, "key size class not built");
  const int dlen = bftq::host_hash_dlen(hash_alg);
  if (dlen == 0) return fail(BFTQ_ERR_INVALID_ARG, "unknown hash algorithm id");
  if (n_items == 0) return BFTQ_OK;
  const KeyView kv = global_keys(e);
  if (!kv.d_keys) return fail(BFTQ_ERR_INVALID_ARG, "no keys registered");
  // Large batches are cut into equal chunks of about host_chunk() items (ArenaRing).
  const uint64_t kChunk = host_chunk();
  const uint64_t n_chunks = n_items <= kChunk + kChunk / 2 ? 1 : (n_items + kChunk - 1) / kChunk;
  const uint64_t per = (n_items + n_chunks - 1) / n_chunks;
  ArenaRing ring{e};
  int rc = BFTQ_OK;
  for (uint64_t c = 0; c < n_chunks && rc == BFTQ_OK; c++) {
    const uint64_t lo = c * per, cnt = std::min(per, n_items - lo);
    Arena& a = ring.next(rc);
    if (rc) break;
    uint8_t *d_sig, *d_dig, *d_st; uint32_t* d_idx;
    a.in(&d_sig, sig_be + lo * key_bytes, (size_t)cnt * key_bytes);
    a.in(&d_dig, digest + lo * dlen, (size_t)cnt * dlen);
    a.in(&d_idx, key_idx + lo, (size_t)cnt);
    a.out(&d_st, out_status + lo, (size_t)cnt);
    rc = a.upload();
    if (rc) break;
    rc = launch_rsa_any(e, kv, d_idx, d_sig, d_dig, hash_alg, cnt, flags, nullptr, d_st, a.stream(), (int)key_bytes);
    if (rc) break;
    rc = a.download_async();
  }
  return ring.drain(rc);
}

// ---- K1b --------------------------------------------------------------------------------------
namespace {
// Per-engine cache of Ed25519 window tables (ed25519_fast.cuh): ONE radix-2^12 table of the base point (5.8 MB, built with the
// cache) and one radix-2^10 table of -A per key (1.7 MB per slot), found by the 32 key bytes.  Slots are immutable once built
// and never move, so kernels of any stream may read them; a table built on one stream is ordered before readers on other
// streams by the build's event.  The cache is bounded (BFTQ_ED25519_CACHE_SLOTS, default 256 = 436 MB): a batch whose new
// keys do not fit runs the table-free kernel.
int ed_build_tables(bftq_engine* e, cudaStream_t st, uint32_t first_slot, uint32_t n_points, bool base_point) {
  namespace ed = bftq::ed;
  EdCache& c = e->ed;
  const int nw = base_point ? ed::FxB::windows : ed::FxA::windows, wbits = base_point ? ed::kFxWB : ed::kFxWA;
  const int multiples = base_point ? ed::FxB::multiples : ed::FxA::multiples;
  ed::gex* d_bases = nullptr;
  CU(cudaMallocAsync((void**)&d_bases, (size_t)n_points * nw * sizeof(ed::gex), st));
  int rc = launch(e, "ed25519_bases_kernel", bftq::ed25519_bases_kernel, grid_per_item(n_points, 32), 32, st, c.d_hdr, first_slot, n_points,
                  d_bases, nw, wbits, base_point ? 1 : 0);
  if (rc) return rc;
  const uint64_t threads = (uint64_t)n_points * nw * (multiples / ed::kFxChunk);
  ed::gea* dst = base_point ? c.d_tabB : c.d_tab + (size_t)first_slot * ed::FxA::entries;
  rc = launch(e, "ed25519_multiples_kernel", bftq::ed25519_multiples_kernel, grid_per_item(threads, 64), 64, st, d_bases, n_points, nw,
              multiples, dst);
  if (rc) return rc;
  CU(cudaFreeAsync(d_bases, st));
  cudaEvent_t ev;
  CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  CU(cudaEventRecord(ev, st));
  c.pending.push_back(ev);
  return BFTQ_OK;
}

int ed_cache_prepare(bftq_engine* e, const uint8_t* pubkeys, uint32_t n_keys, uint64_t max_new, cudaStream_t st, std::vector<uint32_t>& slot_of_key, bool& fits) {
  namespace ed = bftq::ed;
  EdCache& c = e->ed;
  fits = false;
  // which keys are new?
  std::vector<std::string> fresh;
  std::map<std::string, uint32_t> fresh_idx;
  slot_of_key.assign(n_keys, 0);
  for (uint32_t i = 0; i < n_keys; i++) {
    std::string kb((const char*)pubkeys + (size_t)i * 32, 32);
    auto it = c.slot_of.find(kb);
    if (it != c.slot_of.end()) { slot_of_key[i] = it->second; continue; }
    auto f = fresh_idx.find(kb);
    if (f == fresh_idx.end()) { f = fresh_idx.emplace(kb, (uint32_t)fresh.size()).first; fresh.push_back(kb); }
    slot_of_key[i] = 0x80000000u | f->second;                 // resolved below
  }
  if (fresh.size() > max_new) return BFTQ_OK;                  // too few signatures to pay for this many new tables
  if (c.cap_slots == 0) {                                      // first use: the cache itself and the base point's table
    const uint32_t cap = (uint32_t)env_u64("BFTQ_ED25519_CACHE_SLOTS", env_set("BFTQ_ED25519_CACHE_SLOTS") ? 1 : 256);   // set: at least one slot
    void *tab = nullptr, *tabB = nullptr, *hdr = nullptr;
    if (cudaMalloc(&tab, (size_t)cap * ed::FxA::entries * sizeof(ed::gea)) != cudaSuccess ||
        cudaMalloc(&tabB, (size_t)ed::FxB::entries * sizeof(ed::gea)) != cudaSuccess ||
        cudaMalloc(&hdr, (size_t)cap * sizeof(bftq::EdSlotHdr)) != cudaSuccess) {
      cudaGetLastError();                                      // no room: table-free kernel
      if (tab) cudaFree(tab);
      if (tabB) cudaFree(tabB);
      return BFTQ_OK;
    }
    // on the call's stream: a legacy-stream cudaMemset is NOT ordered against the non-blocking streams the builds run on
    // (it raced with the first build's header writes and wiped the 'key decodes' flags: every signature of the first batch invalid)
    if (cudaMemsetAsync(hdr, 0, (size_t)cap * sizeof(bftq::EdSlotHdr), st) != cudaSuccess) { cudaGetLastError(); cudaFree(tab); cudaFree(tabB); cudaFree(hdr); return fail(BFTQ_ERR_CUDA, "cudaMemsetAsync failed"); }
    c.d_tab = (ed::gea*)tab; c.d_tabB = (ed::gea*)tabB; c.d_hdr = (bftq::EdSlotHdr*)hdr; c.cap_slots = cap; c.used = 0;
    const int rc = ed_build_tables(e, st, 0, 1, true);
    if (rc) return rc;
    c.builds += 1;
  }
  const uint32_t n_new = (uint32_t)fresh.size();
  if ((uint64_t)c.used + n_new > c.cap_slots) {
    // Full.  Slots are never evicted one by one (readers of any stream may be using them); a batch that would clearly pay
    // for its tables (128 signatures per new key) and fits an empty cache empties it instead — after the device has drained.
    // Anything smaller takes the table-free kernel, so junk keys cannot make the engine thrash.
    if (n_new > c.cap_slots || max_new < 4ull * n_new) return BFTQ_OK;
    CU(cudaDeviceSynchronize());
    for (cudaEvent_t ev : c.pending) cudaEventDestroy(ev);
    c.pending.clear();
    c.slot_of.clear();
    c.used = 0;
    c.resets++;
    // every key of the call is new now: rebuild the list in first-seen order
    fresh.clear(); fresh_idx.clear();
    for (uint32_t i = 0; i < n_keys; i++) {
      std::string kb((const char*)pubkeys + (size_t)i * 32, 32);
      auto f = fresh_idx.find(kb);
      if (f == fresh_idx.end()) { f = fresh_idx.emplace(kb, (uint32_t)fresh.size()).first; fresh.push_back(kb); }
      slot_of_key[i] = 0x80000000u | f->second;
    }
    if (fresh.size() > c.cap_slots || fresh.size() > max_new) { fits = false; return BFTQ_OK; }
  }
  const uint32_t first = c.used;
  // earlier builds on other streams must be complete before this stream reads their tables
  for (size_t i = 0; i < c.pending.size();) {
    if (cudaEventQuery(c.pending[i]) == cudaSuccess) { cudaEventDestroy(c.pending[i]); c.pending[i] = c.pending.back(); c.pending.pop_back(); }
    else { cudaGetLastError(); CU(cudaStreamWaitEvent(st, c.pending[i], 0)); i++; }
  }
  if (!fresh.empty()) {
    const uint32_t n_build = (uint32_t)fresh.size();
    std::vector<bftq::EdSlotHdr> h(fresh.size());
    for (size_t i = 0; i < fresh.size(); i++) { memset(&h[i], 0, sizeof(h[i])); memcpy(h[i].key, fresh[i].data(), 32); }
    CU(cudaMemcpyAsync(c.d_hdr + first, h.data(), h.size() * sizeof(bftq::EdSlotHdr), cudaMemcpyHostToDevice, st));   // pageable source: staged before return
    const int rc = ed_build_tables(e, st, first, n_build, false);
    if (rc) return rc;
    for (size_t i = 0; i < fresh.size(); i++) c.slot_of.emplace(fresh[i], first + (uint32_t)i);
    c.used = first + n_build;
    c.builds += n_build;
  }
  for (uint32_t i = 0; i < n_keys; i++) if (slot_of_key[i] & 0x80000000u) slot_of_key[i] = c.slot_of[fresh[slot_of_key[i] & 0x7fffffffu]];
  fits = true;
  return BFTQ_OK;
}
}  // namespace

int bftq_ed25519_verify_batch_dev(bftq_engine* e, const uint8_t* pubkeys, uint32_t n_keys, const uint32_t* d_key_idx,
                                  const uint8_t* d_sig, const uint8_t* d_msg, uint64_t n_items, uint8_t* d_status,
                                  void* cuda_stream) {
  if (!e || !pubkeys || !d_key_idx || !d_sig || !d_msg || !d_status) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (n_items == 0) return BFTQ_OK;
  CU(cudaSetDevice(e->device));
  cudaStream_t st = (cudaStream_t)cuda_stream;
  // Signatures run against the cached window tables: at most 48 mixed additions each and no doubling.  A table costs
  // about 1 000 such verifications' worth of work once per key and engine (about 100 table-free ones), so a batch may
  // bring one NEW key per 32 signatures; keys that are cached already cost nothing, whatever the batch size.  Batches
  // with more new keys than that (every signature under its own key, say) take the table-free double-and-add kernel.
  bool tables = e->ed.enabled && n_keys > 0 && n_keys <= 4096;
  if (tables) {
    std::vector<uint32_t> slot_of_key;
    std::lock_guard<std::mutex> g(e->ed.mu);                   // held while this call's work is enqueued
    int rc = ed_cache_prepare(e, pubkeys, n_keys, n_items / 32, st, slot_of_key, tables);
    if (rc) return rc;
    if (tables) {
      const uint64_t n_pad = (n_items + 511) / 512 * 512;
      const size_t xyz_bytes = (size_t)n_pad * 30 * sizeof(int32_t);
      const size_t slot_bytes = ((size_t)n_keys * 4 + 15) / 16 * 16;
      uint8_t* scratch = nullptr;
      CU(cudaMallocAsync((void**)&scratch, xyz_bytes + slot_bytes + n_pad, st));
      int32_t* d_xyz = reinterpret_cast<int32_t*>(scratch);
      uint32_t* d_slot = reinterpret_cast<uint32_t*>(scratch + xyz_bytes);
      uint8_t* d_pre = scratch + xyz_bytes + slot_bytes;
      CU(cudaMemcpyAsync(d_slot, slot_of_key.data(), (size_t)n_keys * 4, cudaMemcpyHostToDevice, st));   // pageable source: staged before return
      rc = launch(e, "ed25519_accumulate_kernel", bftq::ed25519_accumulate_kernel, grid_per_item(n_items, bftq::kEdAccBlock), bftq::kEdAccBlock, st,
                  e->ed.d_tabB, e->ed.d_tab, e->ed.d_hdr, d_slot, n_keys, d_key_idx, d_sig, d_msg, n_items, n_pad, d_xyz, d_pre);
      if (rc) return rc;
      const uint64_t fin_tiles = n_pad / bftq::ed::kFxChunk / bftq::kEdFinBlock;       // one block per 512-item tile of n_pad
      rc = launch(e, "ed25519_finish_kernel", bftq::ed25519_finish_kernel, (unsigned)fin_tiles, bftq::kEdFinBlock, st, d_xyz, d_pre, d_sig,
                  n_items, n_pad, d_status);
      if (rc) return rc;
      CU(cudaFreeAsync(scratch, st));
    }
  }
  if (!tables) {
    uint8_t* d_pk = nullptr;
    CU(cudaMallocAsync((void**)&d_pk, (size_t)std::max<uint32_t>(n_keys, 1) * 32, st));
    if (n_keys) CU(cudaMemcpyAsync(d_pk, pubkeys, (size_t)n_keys * 32, cudaMemcpyHostToDevice, st));
    const int rc = launch(e, "ed25519_verify_kernel", bftq::ed25519_verify_kernel, grid_per_item(n_items, 128), 128, st, d_pk, n_keys, d_key_idx,
                          d_sig, d_msg, n_items, d_status);
    if (rc) return rc;
    CU(cudaFreeAsync(d_pk, st));
  }
  e->stats.items += n_items;
  return BFTQ_OK;
}

int bftq_ed25519_verify_batch(bftq_engine* e, const uint8_t* pubkeys, uint32_t n_keys, const uint32_t* key_idx,
                              const uint8_t* sig, const uint8_t* msg, uint64_t n_items, uint8_t* out_status) {
  if (!e || !pubkeys || !key_idx || !sig || !msg || !out_status) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (n_items == 0) return BFTQ_OK;
  Arena a(e);
  uint8_t *d_sig, *d_msg, *d_st; uint32_t* d_idx;
  a.in(&d_idx, key_idx, (size_t)n_items);
  a.in(&d_sig, sig, (size_t)n_items * 64);
  a.in(&d_msg, msg, (size_t)n_items * 32);
  a.out(&d_st, out_status, (size_t)n_items);
  int rc = a.upload();
  if (rc) return rc;
  rc = bftq_ed25519_verify_batch_dev(e, pubkeys, n_keys, d_idx, d_sig, d_msg, n_items, d_st, a.stream());
  if (rc) return rc;
  return a.download();
}

// ---- K1c --------------------------------------------------------------------------------------
int bftq_ecdsa_p256_verify_batch(bftq_engine* e, const uint8_t* pubkeys, uint32_t n_keys, const uint32_t* key_idx,
                                 const uint8_t* r_be, const uint8_t* s_be, const uint8_t* digest, uint32_t digest_len,
                                 uint64_t n_items, uint8_t* out_status) {
  if (!e || !pubkeys || !key_idx || !r_be || !s_be || !digest || !out_status) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (digest_len == 0 || digest_len > 64) return fail(BFTQ_ERR_INVALID_ARG, "digest_len must be 1..64");
  if (n_items == 0) return BFTQ_OK;
  Arena a(e);
  uint8_t *d_pk, *d_r, *d_s, *d_dg, *d_st; uint32_t* d_idx;
  a.in(&d_pk, pubkeys, (size_t)std::max<uint32_t>(n_keys, 1) * 64, (size_t)n_keys * 64);
  a.in(&d_idx, key_idx, (size_t)n_items);
  a.in(&d_r, r_be, (size_t)n_items * 32);
  a.in(&d_s, s_be, (size_t)n_items * 32);
  a.in(&d_dg, digest, (size_t)n_items * digest_len);
  a.out(&d_st, out_status, (size_t)n_items);
  int rc = a.upload();
  if (rc) return rc;
  rc = launch(e, "ecdsa_p256_verify_kernel", bftq::ecdsa_p256_verify_kernel, grid_per_item(n_items, 128), 128, a.stream(), d_pk, n_keys, d_idx,
              d_r, d_s, d_dg, digest_len, n_items, nullptr, d_st);
  if (rc) return rc;
  e->stats.items += n_items;
  return a.download();
}

// ---- K2 ---------------------------------------------------------------------------------------
}  // extern "C"

struct bftq_quorum {
  bftq::QuorumDev dev;
  uint32_t* d_bits = nullptr;
};

namespace {
int launch_tally(bftq_engine* e, const bftq_quorum* q, const uint32_t* d_off, const uint32_t* d_idx, const uint8_t* d_status,
                 const uint64_t* d_ts, const uint32_t* d_val, uint64_t n_ops, uint32_t* d_winner, uint8_t* d_bits, cudaStream_t st,
                 uint8_t* d_decision = nullptr, uint32_t* d_decided_at = nullptr) {
  const unsigned grid = grid_capped(e, n_ops, 256 / 32, 8);          // one warp per operation
  if (d_ts && d_val)
    return launch(e, "read_tally_kernel", bftq::read_tally_kernel, grid, 256, st, q->dev, d_off, d_idx, d_status, d_ts, d_val, n_ops, d_winner,
                  d_bits, d_decision, d_decided_at);
  return launch(e, "tally_kernel", bftq::tally_kernel, grid, 256, st, q->dev, d_off, d_idx, d_status, n_ops, d_bits);
}
}  // namespace

extern "C" {

int bftq_quorum_create(bftq_engine* e, const bftq_qc_t* qcs, uint32_t n_qc, const uint32_t* member_key_idx,
                       uint32_t n_members, bftq_quorum** out) {
  if (!e || !out || (n_qc && !qcs) || (n_members && !member_key_idx)) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (n_qc > (uint32_t)bftq::kMaxQc) return fail(BFTQ_ERR_INVALID_ARG, "too many quorum cliques");
  uint32_t maxk = 0;
  for (uint32_t c = 0; c < n_qc; c++) {
    if ((uint64_t)qcs[c].member_off + qcs[c].member_cnt > n_members) return fail(BFTQ_ERR_INVALID_ARG, "clique members out of range");
    for (uint32_t m = 0; m < qcs[c].member_cnt; m++) maxk = std::max(maxk, member_key_idx[qcs[c].member_off + m]);
  }
  if (maxk > (1u << 20)) return fail(BFTQ_ERR_INVALID_ARG, "member key index too large");
  auto* q = new bftq_quorum();
  memset(&q->dev, 0, sizeof(q->dev));
  q->dev.nqc = (int32_t)n_qc;
  q->dev.nkeys_words = maxk / 32 + 1;
  std::vector<uint32_t> bits((size_t)std::max<uint32_t>(n_qc, 1) * q->dev.nkeys_words, 0u);
  for (uint32_t c = 0; c < n_qc; c++) {
    q->dev.f[c] = qcs[c].f; q->dev.min[c] = qcs[c].min; q->dev.threshold[c] = qcs[c].threshold; q->dev.suff[c] = qcs[c].suff;
    for (uint32_t m = 0; m < qcs[c].member_cnt; m++) {
      const uint32_t k = member_key_idx[qcs[c].member_off + m];
      bits[(size_t)c * q->dev.nkeys_words + (k >> 5)] |= 1u << (k & 31);
    }
  }
  cudaSetDevice(e->device);
  if (cudaMalloc((void**)&q->d_bits, bits.size() * 4) != cudaSuccess ||
      cudaMemcpy(q->d_bits, bits.data(), bits.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
    delete q;
    return fail(BFTQ_ERR_CUDA, "quorum upload failed");
  }
  q->dev.member_bits = q->d_bits;
  *out = q;
  return BFTQ_OK;
}

void bftq_quorum_destroy(bftq_engine* e, bftq_quorum* q) {
  if (!q) return;
  if (e) cudaSetDevice(e->device);
  if (q->d_bits) { cudaDeviceSynchronize(); cudaFree(q->d_bits); }
  delete q;
}

static int tally_host(bftq_engine* e, const bftq_quorum* q, const uint32_t* op_off, const uint32_t* key_idx, const uint8_t* status,
                      const uint64_t* ts, const uint32_t* value_id, uint64_t n_ops, uint32_t* out_winner, uint8_t* out_bits,
                      uint8_t* out_decision = nullptr, uint32_t* out_decided_at = nullptr) {
  if (!e || !q || !op_off || !out_bits) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (n_ops == 0) return BFTQ_OK;
  const uint64_t n_items = op_off[n_ops];
  if (n_items && (!key_idx || !status)) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (ts && value_id)
    for (uint64_t i = 0; i < n_ops; i++)
      if (op_off[i + 1] - op_off[i] > 32) return fail(BFTQ_ERR_INVALID_ARG, "read tally: more than 32 responders in one operation");
  Arena a(e);
  uint32_t *d_off, *d_idx, *d_val = nullptr, *d_win = nullptr, *d_at = nullptr; uint8_t *d_st, *d_bits, *d_dec = nullptr; uint64_t* d_ts = nullptr;
  a.in(&d_off, op_off, (size_t)n_ops + 1);
  a.in(&d_idx, key_idx, (size_t)std::max<uint64_t>(n_items, 1), (size_t)n_items);
  a.in(&d_st, status, (size_t)std::max<uint64_t>(n_items, 1), (size_t)n_items);
  if (ts && value_id) {
    a.in(&d_ts, ts, (size_t)std::max<uint64_t>(n_items, 1), (size_t)n_items);
    a.in(&d_val, value_id, (size_t)std::max<uint64_t>(n_items, 1), (size_t)n_items);
    a.out(&d_win, out_winner, (size_t)n_ops);
    if (out_decision) { a.out(&d_dec, out_decision, (size_t)n_ops); a.out(&d_at, out_decided_at, (size_t)n_ops); }
  }
  a.out(&d_bits, out_bits, (size_t)n_ops);
  int rc = a.upload();
  if (rc) return rc;
  rc = launch_tally(e, q, d_off, d_idx, d_st, d_ts, d_val, n_ops, d_win, d_bits, a.stream(), d_dec, d_at);
  if (rc) return rc;
  return a.download();
}

int bftq_tally_batch(bftq_engine* e, const bftq_quorum* q, const uint32_t* op_off, const uint32_t* key_idx,
                     const uint8_t* status, uint64_t n_ops, uint8_t* out_bits) {
  return tally_host(e, q, op_off, key_idx, status, nullptr, nullptr, n_ops, nullptr, out_bits);
}

int bftq_read_tally_batch(bftq_engine* e, const bftq_quorum* q, const uint32_t* op_off, const uint32_t* key_idx,
                          const uint8_t* status, const uint64_t* ts, const uint32_t* value_id, uint64_t n_ops,
                          uint32_t* out_winner, uint8_t* out_bits) {
  if (!ts || !value_id || !out_winner) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  return tally_host(e, q, op_off, key_idx, status, ts, value_id, n_ops, out_winner, out_bits);
}

int bftq_read_decide_batch(bftq_engine* e, const bftq_quorum* q, const uint32_t* op_off, const uint32_t* key_idx,
                           const uint8_t* status, const uint64_t* ts, const uint32_t* value_id, uint64_t n_ops,
                           uint8_t* out_decision, uint32_t* out_winner, uint32_t* out_decided_at) {
  if (!ts || !value_id || !out_winner || !out_decision || !out_decided_at) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  std::vector<uint8_t> bits((size_t)std::max<uint64_t>(n_ops, 1));
  return tally_host(e, q, op_off, key_idx, status, ts, value_id, n_ops, out_winner, bits.data(), out_decision, out_decided_at);
}

static int verify_tally_dev_impl(bftq_engine* e, const bftq_quorum* q, const uint32_t* d_op_off, const uint32_t* d_key_idx,
                                 const uint8_t* d_sig_be, const uint8_t* d_digest, uint32_t hash_alg, const uint8_t* d_pre_status,
                                 const uint64_t* d_ts, const uint32_t* d_value_id, uint64_t n_ops, uint64_t n_items, uint32_t flags,
                                 uint8_t* d_status, uint8_t* d_bits, uint32_t* d_winner, uint8_t* d_decision, uint32_t* d_decided_at,
                                 cudaStream_t st) {
  if (!e || !q || !d_op_off || !d_status || !d_bits) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (bftq::host_hash_dlen(hash_alg) == 0) return fail(BFTQ_ERR_INVALID_ARG, "unknown hash algorithm id");
  if (n_ops == 0) return BFTQ_OK;
  CU(cudaSetDevice(e->device));
  if (n_items) {
    int rc = launch_rsa_any(e, global_keys(e), d_key_idx, d_sig_be, d_digest, hash_alg, n_items, flags, d_pre_status, d_status, st);
    if (rc) return rc;
  }
  return launch_tally(e, q, d_op_off, d_key_idx, d_status, d_ts, d_value_id, n_ops, d_winner, d_bits, st, d_decision, d_decided_at);
}

int bftq_verify_tally_batch_dev(bftq_engine* e, const bftq_quorum* q, const uint32_t* d_op_off, const uint32_t* d_key_idx,
                                const uint8_t* d_sig_be, const uint8_t* d_digest, uint32_t hash_alg,
                                const uint8_t* d_pre_status, const uint64_t* d_ts, const uint32_t* d_value_id,
                                uint64_t n_ops, uint64_t n_items, uint32_t flags, uint8_t* d_status, uint8_t* d_bits,
                                uint32_t* d_winner, void* cuda_stream) {
  return verify_tally_dev_impl(e, q, d_op_off, d_key_idx, d_sig_be, d_digest, hash_alg, d_pre_status, d_ts, d_value_id, n_ops, n_items, flags,
                               d_status, d_bits, d_winner, nullptr, nullptr, (cudaStream_t)cuda_stream);
}

int bftq_verify_read_batch_dev(bftq_engine* e, const bftq_quorum* q, const uint32_t* d_op_off, const uint32_t* d_key_idx,
                               const uint8_t* d_sig_be, const uint8_t* d_digest, uint32_t hash_alg, const uint8_t* d_pre_status,
                               const uint64_t* d_ts, const uint32_t* d_value_id, uint64_t n_ops, uint64_t n_items, uint32_t flags,
                               uint8_t* d_status, uint8_t* d_bits, uint8_t* d_decision, uint32_t* d_winner, uint32_t* d_decided_at,
                               void* cuda_stream) {
  if (!d_ts || !d_value_id || !d_decision || !d_winner || !d_decided_at) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  return verify_tally_dev_impl(e, q, d_op_off, d_key_idx, d_sig_be, d_digest, hash_alg, d_pre_status, d_ts, d_value_id, n_ops, n_items, flags,
                               d_status, d_bits, d_winner, d_decision, d_decided_at, (cudaStream_t)cuda_stream);
}

// Host form of the fused verify + tally calls.  The operations are cut into chunks of whole operations (about
// BFTQ_HOST_CHUNK tuples each) that travel through a ring of four staging slots, one stream each: the copies of chunk
// c + 1 run under the kernels of chunk c, pinned caller memory (bftq_host_alloc) is DMA'd in place, pageable memory is
// bounced through the slot's pinned mirror.  The offsets are rebased per chunk in staging.
static int verify_tally_host(bftq_engine* e, const bftq_quorum* q, const uint32_t* op_off, const uint32_t* key_idx, const uint8_t* sig_be,
                             const uint8_t* digest, uint32_t hash_alg, const uint8_t* pre_status, const uint64_t* ts, const uint32_t* value_id,
                             uint64_t n_ops, uint32_t flags, uint8_t* out_status, uint8_t* out_bits, uint32_t* out_winner,
                             uint8_t* out_decision, uint32_t* out_decided_at) {
  if (!e || !q || !op_off || !out_status || !out_bits) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  const int dlen = bftq::host_hash_dlen(hash_alg);
  if (dlen == 0) return fail(BFTQ_ERR_INVALID_ARG, "unknown hash algorithm id");
  if (n_ops == 0) return BFTQ_OK;
  const uint64_t n_items = op_off[n_ops];
  if (n_items && (!key_idx || !sig_be || !digest)) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  const bool read = ts && value_id;
  if (read && !out_winner) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (out_decision && (!read || !out_decided_at)) return fail(BFTQ_ERR_INVALID_ARG, "the read decision needs ts, value_id and out_decided_at");
  for (uint64_t i = 0; i < n_ops; i++) {
    if (op_off[i + 1] < op_off[i]) return fail(BFTQ_ERR_INVALID_ARG, "op_off must be non-decreasing");
    if (read && op_off[i + 1] - op_off[i] > 32) return fail(BFTQ_ERR_INVALID_ARG, "read tally: more than 32 responders in one operation");
  }
  const uint64_t kChunk = host_chunk();
  ArenaRing ring{e};
  int rc = BFTQ_OK;
  uint64_t lo = 0;
  while (lo < n_ops && rc == BFTQ_OK) {
    // chunk [lo, hi): whole operations, about kChunk tuples (at least one operation)
    uint64_t hi = lo + 1;
    if (n_items <= kChunk + kChunk / 2) hi = n_ops;
    else {
      const uint32_t want = op_off[lo] + (uint32_t)std::min<uint64_t>(kChunk, 0xffffffffu - op_off[lo]);
      hi = (uint64_t)(std::upper_bound(op_off + lo + 1, op_off + n_ops + 1, want) - op_off) - 1;
      if (hi <= lo) hi = lo + 1;
      if (n_items - op_off[hi] < kChunk / 2) hi = n_ops;                  // do not leave a sliver behind
    }
    const uint64_t t0 = op_off[lo], cnt = op_off[hi] - t0, nops = hi - lo;
    const size_t ni = (size_t)std::max<uint64_t>(cnt, 1);
    Arena& a = ring.next(rc);
    if (rc) break;
    uint32_t *d_off, *h_off, *d_idx, *d_val = nullptr, *d_win = nullptr, *d_at = nullptr;
    uint8_t *d_sig, *d_dig, *d_pre = nullptr, *d_st, *d_bits, *d_dec = nullptr; uint64_t* d_ts = nullptr;
    a.in(&d_sig, sig_be + t0 * 256, ni * 256, (size_t)cnt * 256);
    a.in(&d_dig, digest + t0 * dlen, ni * dlen, (size_t)cnt * dlen);
    a.in(&d_idx, key_idx + t0, ni, (size_t)cnt);
    if (pre_status) a.in(&d_pre, pre_status + t0, ni, (size_t)cnt);
    if (read) { a.in(&d_ts, ts + t0, ni, (size_t)cnt); a.in(&d_val, value_id + t0, ni, (size_t)cnt); a.out(&d_win, out_winner + lo, (size_t)nops); }
    if (out_decision) { a.out(&d_dec, out_decision + lo, (size_t)nops); a.out(&d_at, out_decided_at + lo, (size_t)nops); }
    a.stage(&d_off, &h_off, (size_t)nops + 1);
    a.out(&d_st, out_status + t0, ni, (size_t)cnt);
    a.out(&d_bits, out_bits + lo, (size_t)nops);
    rc = a.prepare();
    if (rc) break;
    for (uint64_t i = 0; i <= nops; i++) h_off[i] = op_off[lo + i] - (uint32_t)t0;
    rc = a.upload();
    if (rc) break;
    rc = verify_tally_dev_impl(e, q, d_off, d_idx, d_sig, d_dig, hash_alg, d_pre, d_ts, d_val, nops, cnt, flags, d_st, d_bits, d_win, d_dec, d_at,
                               a.stream());
    if (rc) break;
    rc = a.download_async();
    lo = hi;
  }
  return ring.drain(rc);
}

int bftq_verify_tally_batch(bftq_engine* e, const bftq_quorum* q, const uint32_t* op_off, const uint32_t* key_idx,
                            const uint8_t* sig_be, const uint8_t* digest, uint32_t hash_alg, const uint8_t* pre_status,
                            const uint64_t* ts, const uint32_t* value_id, uint64_t n_ops, uint32_t flags,
                            uint8_t* out_status, uint8_t* out_bits, uint32_t* out_winner) {
  return verify_tally_host(e, q, op_off, key_idx, sig_be, digest, hash_alg, pre_status, ts, value_id, n_ops, flags, out_status, out_bits, out_winner,
                           nullptr, nullptr);
}

int bftq_verify_read_batch(bftq_engine* e, const bftq_quorum* q, const uint32_t* op_off, const uint32_t* key_idx, const uint8_t* sig_be,
                           const uint8_t* digest, uint32_t hash_alg, const uint8_t* pre_status, const uint64_t* ts, const uint32_t* value_id,
                           uint64_t n_ops, uint32_t flags, uint8_t* out_status, uint8_t* out_decision, uint32_t* out_winner,
                           uint32_t* out_decided_at) {
  if (!out_decision || !out_winner || !out_decided_at || !ts || !value_id) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  std::vector<uint8_t> bits((size_t)std::max<uint64_t>(n_ops, 1));
  return verify_tally_host(e, q, op_off, key_idx, sig_be, digest, hash_alg, pre_status, ts, value_id, n_ops, flags, out_status, bits.data(), out_winner,
                           out_decision, out_decided_at);
}

// ---- K3 ---------------------------------------------------------------------------------------
}  // extern "C"

namespace {
int check_modulus(const uint8_t* m_be, uint32_t mlen) {
  if (mlen == 0 || mlen > 256) return fail(BFTQ_ERR_INVALID_ARG, "modulus length must be 1..256 bytes");
  if (!(m_be[mlen - 1] & 1)) return fail(BFTQ_ERR_INVALID_ARG, "modulus must be odd");
  bool gt1 = false;
  for (uint32_t i = 0; i + 1 < mlen; i++) gt1 = gt1 || m_be[i];
  if (!gt1 && m_be[mlen - 1] <= 1) return fail(BFTQ_ERR_INVALID_ARG, "modulus must be > 1");
  return BFTQ_OK;
}

// lambda / combine launcher on an existing arena stream (device pointers).
template <int L>
int launch_lagrange(bftq_engine* e, const uint8_t* m_be, uint32_t mlen, uint32_t k, const int32_t* d_x, const uint8_t* d_y, uint64_t n_items,
                    uint8_t* d_out, uint8_t* d_st, uint8_t* d_lambda, cudaStream_t st) {
  bftq::LagrangeMod<L> M;
  bftq::make_lagrange_mod<L>(m_be, mlen, M);
  return launch(e, "lagrange_combine_kernel", bftq::lagrange_combine_kernel<L>, grid_per_item(n_items, 128), 128, st, M, k, d_x, d_y, n_items,
                d_out, d_st, d_lambda);
}
int launch_lagrange_any(bftq_engine* e, const uint8_t* m_be, uint32_t mlen, uint32_t k, const int32_t* d_x, const uint8_t* d_y,
                        uint64_t n_items, uint8_t* d_out, uint8_t* d_st, uint8_t* d_lambda, cudaStream_t st) {
  if (mlen <= 32) return launch_lagrange<8>(e, m_be, mlen, k, d_x, d_y, n_items, d_out, d_st, d_lambda, st);
  if (mlen <= 64) return launch_lagrange<16>(e, m_be, mlen, k, d_x, d_y, n_items, d_out, d_st, d_lambda, st);
  if (mlen <= 128) return launch_lagrange<32>(e, m_be, mlen, k, d_x, d_y, n_items, d_out, d_st, d_lambda, st);
  return launch_lagrange<64>(e, m_be, mlen, k, d_x, d_y, n_items, d_out, d_st, d_lambda, st);
}

// ---- K5 plumbing ---------------------------------------------------------------------------------
template <int W>
int make_moddev(const uint8_t* p_be, uint32_t plen, bftq::ModDev<W>& M) {
  if (plen != 16u * W) return fail(BFTQ_ERR_INVALID_ARG, "internal: modulus class mismatch");
  UBig n;
  from_be(n, p_be, plen);
  if (bitlen(n) != 128 * W || !(n.w[0] & 1)) return fail(BFTQ_ERR_UNSUPPORTED_KEY, "exponentiation modulus must be odd with exactly 8*len bits");
  memset(&M, 0, sizeof(M));
  to_words(n, M.n, 4 * W);
  M.n0inv = neg_inv32(M.n[0]);
  M.nbytes = plen;
  UBig one;
  memset(&one, 0, sizeof(one));
  one.w[0] = 1;
  to_words(shl_mod(one, n, 2 * 128 * W), M.r2, 4 * W);
  return BFTQ_OK;
}
template <int W>
int launch_modexp(bftq_engine* e, const uint8_t* p_be, uint32_t plen, const uint8_t* d_base, const uint8_t* d_exp, uint32_t elen, uint64_t n,
                  uint8_t* d_out, cudaStream_t st, uint32_t n_bases = 0) {
  bftq::ModDev<W> M;
  int rc = make_moddev<W>(p_be, plen, M);
  if (rc) return rc;
  return launch(e, "modexp_kernel", bftq::modexp_kernel<W, 128>, grid_capped(e, n, 4 * 8, 4), 128, st, M, d_base, d_exp, elen, n, d_out, n_bases);
}
template <int W>
int launch_modprod(bftq_engine* e, const uint8_t* p_be, uint32_t plen, const uint8_t* d_vals, uint32_t k, uint64_t n, uint8_t* d_out, cudaStream_t st) {
  bftq::ModDev<W> M;
  int rc = make_moddev<W>(p_be, plen, M);
  if (rc) return rc;
  return launch(e, "modprod_kernel", bftq::modprod_kernel<W, 128>, grid_capped(e, n, 4 * 8, 4), 128, st, M, d_vals, k, n, d_out);
}
int modexp_any(bftq_engine* e, const uint8_t* p_be, uint32_t plen, const uint8_t* d_base, const uint8_t* d_exp, uint32_t elen, uint64_t n,
               uint8_t* d_out, cudaStream_t st, uint32_t n_bases = 0) {
  if (plen == 128) return launch_modexp<8>(e, p_be, plen, d_base, d_exp, elen, n, d_out, st, n_bases);
  if (plen == 256) return launch_modexp<16>(e, p_be, plen, d_base, d_exp, elen, n, d_out, st, n_bases);
  return fail(BFTQ_ERR_UNSUPPORTED_KEY, "exponentiation modulus must be 128 or 256 bytes (1024 / 2048 bit)");
}
int modprod_any(bftq_engine* e, const uint8_t* p_be, uint32_t plen, const uint8_t* d_vals, uint32_t k, uint64_t n, uint8_t* d_out, cudaStream_t st) {
  if (plen == 128) return launch_modprod<8>(e, p_be, plen, d_vals, k, n, d_out, st);
  if (plen == 256) return launch_modprod<16>(e, p_be, plen, d_vals, k, n, d_out, st);
  return fail(BFTQ_ERR_UNSUPPORTED_KEY, "exponentiation modulus must be 128 or 256 bytes (1024 / 2048 bit)");
}
}  // namespace

extern "C" {

int bftq_lagrange_combine_batch(bftq_engine* e, const uint8_t* m_be, uint32_t mlen, uint32_t k, const int32_t* x,
                                const uint8_t* y_be, uint64_t n_items, uint8_t* out_be, uint8_t* out_status) {
  if (!e || !m_be || !x || !y_be || !out_be || !out_status) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (k == 0 || k > 255) return fail(BFTQ_ERR_INVALID_ARG, "k must be 1..255");
  int rc = check_modulus(m_be, mlen);
  if (rc) return rc;
  if (n_items == 0) return BFTQ_OK;
  Arena a(e);
  int32_t* d_x; uint8_t *d_y, *d_out, *d_st;
  a.in(&d_x, x, (size_t)n_items * k);
  a.in(&d_y, y_be, (size_t)n_items * k * mlen);
  a.out(&d_out, out_be, (size_t)n_items * mlen);
  a.out(&d_st, out_status, (size_t)n_items);
  rc = a.upload();
  if (rc) return rc;
  rc = launch_lagrange_any(e, m_be, mlen, k, d_x, d_y, n_items, d_out, d_st, nullptr, a.stream());
  if (rc) return rc;
  return a.download();
}

int bftq_lagrange_combine_batch_dev(bftq_engine* e, const uint8_t* m_be, uint32_t mlen, uint32_t k, const int32_t* d_x, const uint8_t* d_y_be,
                                    uint64_t n_items, uint8_t* d_out_be, uint8_t* d_status, void* cuda_stream) {
  if (!e || !m_be || !d_x || !d_y_be || !d_out_be || !d_status) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (k == 0 || k > 255) return fail(BFTQ_ERR_INVALID_ARG, "k must be 1..255");
  int rc = check_modulus(m_be, mlen);
  if (rc) return rc;
  if (n_items == 0) return BFTQ_OK;
  CU(cudaSetDevice(e->device));
  return launch_lagrange_any(e, m_be, mlen, k, d_x, d_y_be, n_items, d_out_be, d_status, nullptr, (cudaStream_t)cuda_stream);
}

// ---- K5 ---------------------------------------------------------------------------------------
int bftq_modexp_batch(bftq_engine* e, const uint8_t* m_be, uint32_t mlen, const uint8_t* base_be, const uint8_t* exp_be, uint32_t elen,
                      uint64_t n_items, uint8_t* out_be) {
  if (!e || !m_be || !base_be || !exp_be || !out_be || elen == 0) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (n_items == 0) return BFTQ_OK;
  Arena a(e);
  uint8_t *d_b, *d_e, *d_o;
  a.in(&d_b, base_be, (size_t)n_items * mlen);
  a.in(&d_e, exp_be, (size_t)n_items * elen);
  a.out(&d_o, out_be, (size_t)n_items * mlen);
  int rc = a.upload();
  if (rc) return rc;
  rc = modexp_any(e, m_be, mlen, d_b, d_e, elen, n_items, d_o, a.stream());
  if (rc) return rc;
  return a.download();
}

int bftq_modprod_batch(bftq_engine* e, const uint8_t* m_be, uint32_t mlen, uint32_t k, const uint8_t* vals_be, uint64_t n_items,
                       uint8_t* out_be) {
  if (!e || !m_be || !vals_be || !out_be || k == 0) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (n_items == 0) return BFTQ_OK;
  Arena a(e);
  uint8_t *d_v, *d_o;
  a.in(&d_v, vals_be, (size_t)n_items * k * mlen);
  a.out(&d_o, out_be, (size_t)n_items * mlen);
  int rc = a.upload();
  if (rc) return rc;
  rc = modprod_any(e, m_be, mlen, d_v, k, n_items, d_o, a.stream());
  if (rc) return rc;
  return a.download();
}

}  // extern "C"
namespace {
// prod_i Y_i^lambda_i mod p with lambda_i = Lagrange(x_i, xs, q): K3 (lambda) -> K5 modexp -> K5 product.
int lagrange_exp_product_dev(bftq_engine* e, cudaStream_t st, const uint8_t* p_be, uint32_t plen, const uint8_t* q_be, uint32_t qlen, uint32_t k,
                             const int32_t* d_x, const uint8_t* d_y, uint64_t n_items, uint8_t* d_lambda, uint8_t* d_pow, uint8_t* d_dummy_out,
                             uint8_t* d_st, uint8_t* d_prod) {
  // lambda only: feed the combine kernel zero shares (d_pow is zero-initialised scratch of sufficient size is not
  // needed: y is read but its product is discarded) — reuse d_y's first bytes as y is only multiplied in.
  int rc = launch_lagrange_any(e, q_be, qlen, k, d_x, d_lambda /* any readable k*qlen bytes per item */, n_items, d_dummy_out, d_st, d_lambda, st);
  if (rc) return rc;
  rc = modexp_any(e, p_be, plen, d_y, d_lambda, qlen, n_items * k, d_pow, st);
  if (rc) return rc;
  return modprod_any(e, p_be, plen, d_pow, k, n_items, d_prod, st);
}

// CalculateR's device scratch for n items of k shares, declared on the call's arena.
struct DsaRScratch {
  uint8_t *lam, *pow, *tmp, *prod, *v, *vinv, *rp, *st2;
  void declare(Arena& a, uint64_t n, uint32_t k, uint32_t plen, uint32_t qlen) {
    a.out(&lam, (uint8_t*)nullptr, (size_t)n * k * qlen, 0);
    a.out(&pow, (uint8_t*)nullptr, (size_t)n * k * plen, 0);
    a.out(&tmp, (uint8_t*)nullptr, (size_t)n * qlen, 0);
    a.out(&prod, (uint8_t*)nullptr, (size_t)n * plen, 0);
    a.out(&v, (uint8_t*)nullptr, (size_t)n * qlen, 0);
    a.out(&vinv, (uint8_t*)nullptr, (size_t)n * qlen, 0);
    a.out(&rp, (uint8_t*)nullptr, (size_t)n * plen, 0);
    a.out(&st2, (uint8_t*)nullptr, (size_t)n, 0);
  }
};
// dsaGroupOperations.CalculateR over one group (dsa.go:33-52), device pointers: d_ri n x k x plen (< p), d_vi n x k x qlen,
// d_out n x qlen, d_st n.  go_inverse: the exponent is Go's v.ModInverse(v, q) (thdsa_go_inverse_kernel: v^-1, or v when
// there is none); otherwise Fermat's v^(q-2) with status 3 for v = 0 (q prime).  Status 3 also marks a lambda whose
// denominator has no inverse mod q.
int dsa_calculate_r_dev(bftq_engine* e, cudaStream_t st, const uint8_t* p_be, uint32_t plen, const uint8_t* q_be, uint32_t qlen, uint32_t k,
                        const int32_t* d_x, const uint8_t* d_ri, const uint8_t* d_vi, uint64_t n_items, const DsaRScratch& s, bool go_inverse,
                        uint8_t* d_out, uint8_t* d_st) {
  CU(cudaMemsetAsync(s.lam, 0, (size_t)n_items * k * qlen, st));
  // r' = prod R_i^lambda_i mod p                                    (dsa.go:41-46)
  int rc = lagrange_exp_product_dev(e, st, p_be, plen, q_be, qlen, k, d_x, d_ri, n_items, s.lam, s.pow, s.tmp, d_st, s.prod);
  if (rc) return rc;
  // v = sum v_i lambda_i mod q                                      (dsa.go:47-48)
  rc = launch_lagrange_any(e, q_be, qlen, k, d_x, d_vi, n_items, s.v, s.st2, nullptr, st);
  if (rc) return rc;
  // v^-1 mod q                                                      (dsa.go:49)
  bftq::LagrangeMod<8> M;
  bftq::make_lagrange_mod<8>(q_be, qlen, M);
  if (go_inverse) rc = launch(e, "thdsa_go_inverse_kernel", bftq::thdsa_go_inverse_kernel<8>, grid_per_item(n_items, 128), 128, st, M, s.v, n_items, s.vinv);
  else rc = launch(e, "fermat_inverse_kernel", bftq::fermat_inverse_kernel<8>, grid_per_item(n_items, 128), 128, st, M, s.v, n_items, s.vinv, d_st);
  if (rc) return rc;
  // r = r'^(v^-1) mod p                                             (dsa.go:50)
  rc = modexp_any(e, p_be, plen, s.prod, s.vinv, qlen, n_items, s.rp, st);
  if (rc) return rc;
  // r mod q                                                         (dsa.go:51)
  return launch(e, "mod_small_kernel", bftq::mod_small_kernel<8>, grid_per_item(n_items, 128), 128, st, M, s.rp, plen, n_items, d_out);
}

struct EcdsaRScratch {
  uint8_t *lam, *tmp, *v, *vinv, *ok, *st2;
  uint32_t* jac;
  void declare(Arena& a, uint64_t n, uint32_t k) {
    a.out(&lam, (uint8_t*)nullptr, (size_t)n * k * 32, 0);
    a.out(&tmp, (uint8_t*)nullptr, (size_t)n * 32, 0);
    a.out(&v, (uint8_t*)nullptr, (size_t)n * 32, 0);
    a.out(&vinv, (uint8_t*)nullptr, (size_t)n * 32, 0);
    a.out(&jac, (uint32_t*)nullptr, (size_t)n * k * 24, 0);
    a.out(&ok, (uint8_t*)nullptr, (size_t)n * k, 0);
    a.out(&st2, (uint8_t*)nullptr, (size_t)n, 0);
  }
};
// ecdsaGroupOperations.CalculateR on P-256 (ecdsa.go:36-59), device pointers: d_ri n x k x 65, d_vi n x k x 32, d_out n x 32,
// d_st n: 3 where an R_i is not a curve point or the result is at infinity (r = 0 there).  N is prime, so Fermat's inverse
// is Go's ModInverse, and v = 0 gives v^-1 = 0, r = 0 as Go's.
int ecdsa_calculate_r_dev(bftq_engine* e, cudaStream_t st, uint32_t k, const int32_t* d_x, const uint8_t* d_ri, const uint8_t* d_vi, uint64_t n_items,
                          const EcdsaRScratch& s, uint8_t* d_out, uint8_t* d_st) {
  CU(cudaMemsetAsync(s.lam, 0, (size_t)n_items * k * 32, st));
  int rc = launch_lagrange_any(e, kP256N, 32, k, d_x, s.lam, n_items, s.tmp, s.st2, s.lam, st);        // lambda_i mod N
  if (rc) return rc;
  rc = launch(e, "p256_scalar_mul_kernel", bftq::p256_scalar_mul_kernel, grid_per_item(n_items * k, 128), 128, st, d_ri, s.lam, n_items * k,
              s.jac, s.ok);
  if (rc) return rc;
  rc = launch_lagrange_any(e, kP256N, 32, k, d_x, d_vi, n_items, s.v, s.st2, nullptr, st);           // v = sum v_i lambda_i
  if (rc) return rc;
  bftq::LagrangeMod<8> M;
  bftq::make_lagrange_mod<8>(kP256N, 32, M);
  rc = launch(e, "fermat_inverse_kernel", bftq::fermat_inverse_kernel<8>, grid_per_item(n_items, 128), 128, st, M, s.v, n_items, s.vinv, nullptr);
  if (rc) return rc;
  return launch(e, "p256_sum_mul_kernel", bftq::p256_sum_mul_kernel, grid_per_item(n_items, 128), 128, st, s.jac, s.ok, k, s.vinv, n_items, d_out,
                d_st);
}
}  // namespace
extern "C" {

int bftq_lagrange_exp_product_batch(bftq_engine* e, const uint8_t* p_be, uint32_t plen, const uint8_t* q_be, uint32_t qlen, uint32_t k,
                                    const int32_t* x, const uint8_t* y_be, uint64_t n_items, uint8_t* out_be, uint8_t* out_status) {
  if (!e || !p_be || !q_be || !x || !y_be || !out_be || !out_status) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (k == 0 || k > 255) return fail(BFTQ_ERR_INVALID_ARG, "k must be 1..255");
  int rc = check_modulus(q_be, qlen);
  if (rc) return rc;
  if (n_items == 0) return BFTQ_OK;
  Arena a(e);
  int32_t* d_x; uint8_t *d_y, *d_lam, *d_pow, *d_tmp, *d_st, *d_out;
  a.in(&d_x, x, (size_t)n_items * k);
  a.in(&d_y, y_be, (size_t)n_items * k * plen);
  a.out(&d_lam, (uint8_t*)nullptr, (size_t)n_items * k * qlen, 0);
  a.out(&d_pow, (uint8_t*)nullptr, (size_t)n_items * k * plen, 0);
  a.out(&d_tmp, (uint8_t*)nullptr, (size_t)n_items * qlen, 0);
  a.out(&d_st, out_status, (size_t)n_items);
  a.out(&d_out, out_be, (size_t)n_items * plen);
  rc = a.upload();
  if (rc) return rc;
  CU(cudaMemsetAsync(d_lam, 0, (size_t)n_items * k * qlen, a.stream()));
  rc = lagrange_exp_product_dev(e, a.stream(), p_be, plen, q_be, qlen, k, d_x, d_y, n_items, d_lam, d_pow, d_tmp, d_st, d_out);
  if (rc) return rc;
  return a.download();
}

int bftq_dsa_calculate_r_batch(bftq_engine* e, const uint8_t* p_be, uint32_t plen, const uint8_t* q_be, uint32_t qlen, uint32_t k,
                               const int32_t* x, const uint8_t* ri_be, const uint8_t* vi_be, uint64_t n_items, uint8_t* out_r_be,
                               uint8_t* out_status) {
  if (!e || !p_be || !q_be || !x || !ri_be || !vi_be || !out_r_be || !out_status) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (k == 0 || k > 255) return fail(BFTQ_ERR_INVALID_ARG, "k must be 1..255");
  if (qlen > 32) return fail(BFTQ_ERR_UNSUPPORTED_KEY, "subgroup order longer than 256 bits");
  int rc = check_modulus(q_be, qlen);
  if (rc) return rc;
  if (n_items == 0) return BFTQ_OK;
  Arena a(e);
  int32_t* d_x; uint8_t *d_ri, *d_vi, *d_st, *d_out;
  DsaRScratch s;
  a.in(&d_x, x, (size_t)n_items * k);
  a.in(&d_ri, ri_be, (size_t)n_items * k * plen);
  a.in(&d_vi, vi_be, (size_t)n_items * k * qlen);
  s.declare(a, n_items, k, plen, qlen);
  a.out(&d_st, out_status, (size_t)n_items);
  a.out(&d_out, out_r_be, (size_t)n_items * qlen);
  rc = a.upload();
  if (rc) return rc;
  rc = dsa_calculate_r_dev(e, a.stream(), p_be, plen, q_be, qlen, k, d_x, d_ri, d_vi, n_items, s, false, d_out, d_st);
  if (rc) return rc;
  return a.download();
}

int bftq_ecdsa_p256_calculate_r_batch(bftq_engine* e, uint32_t k, const int32_t* x, const uint8_t* ri, const uint8_t* vi_be,
                                      uint64_t n_items, uint8_t* out_r_be, uint8_t* out_status) {
  if (!e || !x || !ri || !vi_be || !out_r_be || !out_status) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (k == 0 || k > 255) return fail(BFTQ_ERR_INVALID_ARG, "k must be 1..255");
  if (n_items == 0) return BFTQ_OK;
  Arena a(e);
  int32_t* d_x; uint8_t *d_ri, *d_vi, *d_st, *d_out;
  EcdsaRScratch s;
  a.in(&d_x, x, (size_t)n_items * k);
  a.in(&d_ri, ri, (size_t)n_items * k * 65);
  a.in(&d_vi, vi_be, (size_t)n_items * k * 32);
  s.declare(a, n_items, k);
  a.out(&d_st, out_status, (size_t)n_items);
  a.out(&d_out, out_r_be, (size_t)n_items * 32);
  int rc = a.upload();
  if (rc) return rc;
  rc = ecdsa_calculate_r_dev(e, a.stream(), k, d_x, d_ri, d_vi, n_items, s, d_out, d_st);
  if (rc) return rc;
  return a.download();
}

// ---- K1d: DSA verify ----------------------------------------------------------------------------
}  // extern "C"
namespace {
// Domain check for one DSA key: p odd with exactly 1024 / 2048 bits (K5's classes), q odd, at most 256 bits.
// Returns 0 usable, 1 dsa.Verify is false for every signature (q's bit length is not a multiple of 8), 2 not built.
int dsa_key_class(const uint8_t* p_be, uint32_t plen, const uint8_t* q_be, uint32_t qlen) {
  if (!(plen == 128 || plen == 256) || qlen == 0 || qlen > 32) return 2;
  if (!(p_be[0] & 0x80) || !(p_be[plen - 1] & 1) || !(q_be[qlen - 1] & 1)) return 2;
  if (!(q_be[0] & 0x80)) return q_be[0] == 0 ? 2 : 1;
  return 0;
}
// d_r / d_s: 32-byte right-aligned values `stride` apart; d_bases: g || y (2 x plen); scratch: d_u (2n x qlen),
// d_pow (2n x plen), d_prod (n x plen).  d_pre may be NULL.
int dsa_verify_dev(bftq_engine* e, const uint8_t* p_be, uint32_t plen, const uint8_t* q_be, uint32_t qlen, const uint8_t* d_bases,
                   const uint8_t* d_r, const uint8_t* d_s, uint32_t stride, const uint8_t* d_dig, uint32_t dlen, uint64_t n,
                   const uint8_t* d_pre, uint8_t* d_u, uint8_t* d_pow, uint8_t* d_prod, uint8_t* d_st, cudaStream_t st) {
  bftq::LagrangeMod<8> M;
  bftq::make_lagrange_mod<8>(q_be, qlen, M);
  int rc = launch(e, "dsa_prepare_kernel", bftq::dsa_prepare_kernel<8>, grid_per_item(n, 128), 128, st, M, d_r, d_s, stride, d_dig, dlen, n,
                  d_pre, d_u, d_st);
  if (rc) return rc;
  rc = modexp_any(e, p_be, plen, d_bases, d_u, qlen, 2 * n, d_pow, st, 2);
  if (rc) return rc;
  rc = modprod_any(e, p_be, plen, d_pow, 2, n, d_prod, st);
  if (rc) return rc;
  rc = launch(e, "dsa_finish_kernel", bftq::dsa_finish_kernel<8>, grid_per_item(n, 128), 128, st, M, d_prod, plen, d_r, stride, n, d_st);
  if (rc) return rc;
  e->stats.items += n;
  return BFTQ_OK;
}
}  // namespace
extern "C" {

int bftq_dsa_verify_batch(bftq_engine* e, const uint8_t* p_be, uint32_t plen, const uint8_t* q_be, uint32_t qlen, const uint8_t* g_be,
                          const uint8_t* y_be, const uint8_t* r_be, const uint8_t* s_be, const uint8_t* digest, uint32_t digest_len,
                          uint64_t n_items, uint8_t* out_status) {
  if (!e || !p_be || !q_be || !g_be || !y_be || !r_be || !s_be || !digest || !out_status) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (digest_len == 0 || digest_len > 64) return fail(BFTQ_ERR_INVALID_ARG, "digest_len must be 1..64");
  const int cls = dsa_key_class(p_be, plen, q_be, qlen);
  if (cls == 2) return fail(BFTQ_ERR_UNSUPPORTED_KEY, "DSA domain: p must be odd with exactly 1024 / 2048 bits in plen bytes, q odd of at most 256 bits");
  if (n_items == 0) return BFTQ_OK;
  if (cls == 1) { memset(out_status, BFTQ_ST_BAD_SIGNATURE, (size_t)n_items); return BFTQ_OK; }   // dsa.Verify: q.BitLen() & 7 != 0
  std::vector<uint8_t> bases(2 * (size_t)plen);
  memcpy(bases.data(), g_be, plen);
  memcpy(bases.data() + plen, y_be, plen);
  Arena a(e);
  uint8_t *d_b, *d_r, *d_s, *d_dg, *d_u, *d_pow, *d_prod, *d_st;
  a.in(&d_b, bases.data(), bases.size());
  a.in(&d_r, r_be, (size_t)n_items * 32);
  a.in(&d_s, s_be, (size_t)n_items * 32);
  a.in(&d_dg, digest, (size_t)n_items * digest_len);
  a.out(&d_u, (uint8_t*)nullptr, 2 * (size_t)n_items * qlen, 0);
  a.out(&d_pow, (uint8_t*)nullptr, 2 * (size_t)n_items * plen, 0);
  a.out(&d_prod, (uint8_t*)nullptr, (size_t)n_items * plen, 0);
  a.out(&d_st, out_status, (size_t)n_items);
  int rc = a.upload();
  if (rc) return rc;
  rc = dsa_verify_dev(e, p_be, plen, q_be, qlen, d_b, d_r, d_s, 32, d_dg, digest_len, n_items, nullptr, d_u, d_pow, d_prod, d_st, a.stream());
  if (rc) return rc;
  return a.download();
}

// ---- K4 ---------------------------------------------------------------------------------------
int bftq_pgp_digest_batch(bftq_engine* e, const uint8_t* data_blob, const uint64_t* data_off, uint32_t n_data,
                          const uint32_t* data_idx, const uint8_t* suffix_blob, const uint64_t* suffix_off,
                          uint32_t hash_alg, uint64_t n_items, uint8_t* out_digest) {
  if (!e || !data_off || !suffix_off || !out_digest) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  if (!bftq::digest_on_device(hash_alg)) return fail(BFTQ_ERR_INVALID_ARG, "digest algorithm not built for the device (SHA-1/224/256/384/512 are)");
  const int dlen = bftq::host_hash_dlen(hash_alg);
  if (n_items == 0) return BFTQ_OK;
  if (!data_idx && n_data < n_items) return fail(BFTQ_ERR_INVALID_ARG, "data_idx is NULL but n_data < n_items");
  if (data_idx)
    for (uint64_t i = 0; i < n_items; i++)
      if (data_idx[i] >= n_data) return fail(BFTQ_ERR_INVALID_ARG, "data_idx out of range");
  const size_t dbytes = (size_t)data_off[n_data], sbytes = (size_t)suffix_off[n_items];
  if ((dbytes && !data_blob) || (sbytes && !suffix_blob)) return fail(BFTQ_ERR_INVALID_ARG, "NULL blob");
  Arena a(e);
  uint8_t *d_data, *d_suf, *d_out; uint64_t *d_doff, *d_soff; uint32_t* d_didx = nullptr;
  a.in(&d_data, data_blob, std::max<size_t>(dbytes, 1), dbytes);
  a.in(&d_suf, suffix_blob, std::max<size_t>(sbytes, 1), sbytes);
  a.in(&d_doff, data_off, (size_t)n_data + 1);
  a.in(&d_soff, suffix_off, (size_t)n_items + 1);
  if (data_idx) a.in(&d_didx, data_idx, (size_t)n_items);
  a.out(&d_out, out_digest, (size_t)n_items * dlen);
  int rc = a.upload();
  if (rc) return rc;
  rc = launch(e, "pgp_digest_kernel", bftq::pgp_digest_kernel_for(hash_alg), grid_per_item(n_items, 128), 128, a.stream(), d_data, d_doff, d_didx,
              d_suf, d_soff, n_items, d_out, nullptr, nullptr);
  if (rc) return rc;
  return a.download();
}

// ---- host packer ------------------------------------------------------------------------------
}  // extern "C"
#include "packer_host.inc"
#include "decrypt_host.inc"
#include "thrsa_host.inc"
#include "thdsa_host.inc"
#include "auth_host.inc"
#include "auth_client_host.inc"
#include "thdsa_proc_host.inc"
#include "data_host.inc"

extern "C" {
// After the .inc files: the handle lists detach handle types defined there.
void bftq_shutdown(bftq_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  e->keyrings.shutdown();
  e->thrsa.shutdown();
  e->thdsa.shutdown();
  e->auth.shutdown();
  e->auth_client.shutdown();
  for (auto& kv : e->host_allocs) cudaFreeHost(kv.first);
  for (auto* s : e->slots) {
    if (s->stream) { cudaStreamSynchronize(s->stream); cudaStreamDestroy(s->stream); }
    if (s->done) cudaEventDestroy(s->done);
    if (s->h_pinned) cudaFreeHost(s->h_pinned);
    if (s->d_buf) cudaFree(s->d_buf);
    delete s;
  }
  if (e->d_keys) cudaFree(e->d_keys);
  if (e->d_keys32) cudaFree(e->d_keys32);
  if (e->d_p256_base) cudaFree(e->d_p256_base);
  if (e->d_auth_group) cudaFree(e->d_auth_group);
  if (e->d_auth_group_q) cudaFree(e->d_auth_group_q);
  cudaDeviceSynchronize();
  for (auto& b : e->scratch.free_list) cudaFree(b.first);
  for (cudaEvent_t ev : e->ed.pending) cudaEventDestroy(ev);
  if (e->ed.d_tab) cudaFree(e->ed.d_tab);
  if (e->ed.d_tabB) cudaFree(e->ed.d_tabB);
  if (e->ed.d_hdr) cudaFree(e->ed.d_hdr);
  for (void* p : e->retired) cudaFree(p);
  delete e;
}
}  // extern "C"

// ---- quorum-descriptor builder ------------------------------------------------------------------
// The descriptor the reference recomputes on EVERY call (client.go:64,101,141,238; server.go:182,211,237,300,473) is a
// function of the trust graph alone: it is cached per rw flag set and stamped with the graph's version, which every
// mutation (AddNodes / SetSelfNodes / RemoveNodes / Revoke — certificate revocation included, graph.go:131-146) advances.
struct bftq_graph {
  std::mutex mu;
  bftq::wot::Graph g;
  uint64_t version = 1;
  std::map<int, std::pair<uint64_t, std::vector<bftq::wot::QC>>> cache;      // rw -> (version it was built at, cliques)
  uint64_t hits = 0, builds = 0;
};
extern "C" {
int bftq_graph_create(bftq_graph** out) {
  if (!out) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  *out = new bftq_graph();
  return BFTQ_OK;
}
void bftq_graph_destroy(bftq_graph* g) { delete g; }
int bftq_graph_add_node(bftq_graph* g, uint64_t id, const uint64_t* signer_ids, uint32_t n_signers) {
  if (!g || (n_signers && !signer_ids)) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  std::lock_guard<std::mutex> l(g->mu);
  g->g.add_node(id, signer_ids, n_signers);
  g->version++;
  return BFTQ_OK;
}
int bftq_graph_set_self(bftq_graph* g, uint64_t id) {
  if (!g) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  std::lock_guard<std::mutex> l(g->mu);
  g->g.set_self(id);
  g->version++;
  return BFTQ_OK;
}
int bftq_graph_remove_node(bftq_graph* g, uint64_t id) {
  if (!g) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  std::lock_guard<std::mutex> l(g->mu);
  g->g.remove_node(id);
  g->version++;
  return BFTQ_OK;
}
int bftq_graph_revoke(bftq_graph* g, uint64_t id) {
  if (!g) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  std::lock_guard<std::mutex> l(g->mu);
  g->g.revoke(id);
  g->version++;
  return BFTQ_OK;
}
int bftq_graph_version(bftq_graph* g, uint64_t* version, uint64_t* cache_hits, uint64_t* cache_builds) {
  if (!g || !version) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  std::lock_guard<std::mutex> l(g->mu);
  *version = g->version;
  if (cache_hits) *cache_hits = g->hits;
  if (cache_builds) *cache_builds = g->builds;
  return BFTQ_OK;
}
int bftq_graph_choose_quorum(bftq_graph* g, int rw, bftq_qc_ids_t* out_qcs, uint32_t cap_qc, uint32_t* n_qc, uint64_t* out_members,
                             uint32_t cap_members, uint32_t* n_members) {
  if (!g || !n_qc || !n_members) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  std::vector<bftq::wot::QC> qcs;
  {
    std::lock_guard<std::mutex> l(g->mu);
    auto it = g->cache.find(rw);
    if (it != g->cache.end() && it->second.first == g->version) { qcs = it->second.second; g->hits++; }
    else {
      g->g.choose_quorum(rw, qcs);
      g->cache[rw] = std::make_pair(g->version, qcs);
      g->builds++;
    }
  }
  uint32_t off = 0;
  for (size_t c = 0; c < qcs.size(); c++) {
    if (out_qcs && c < cap_qc) out_qcs[c] = bftq_qc_ids_t{qcs[c].f, qcs[c].min, qcs[c].threshold, qcs[c].suff, off, (uint32_t)qcs[c].nodes.size()};
    for (uint64_t id : qcs[c].nodes) { if (out_members && off < cap_members) out_members[off] = id; off++; }
  }
  *n_qc = (uint32_t)qcs.size();
  *n_members = off;
  return BFTQ_OK;
}

// Client.revoke's scan (protocol/client.go:304-346), batched: per operation, the signers (Signers(ss) of every good
// response, in bucket order) that appear under two DIFFERENT values at the same timestamp t > 0.  A signer is remembered
// under the first value it is seen with (dup_map[id] gets exactly one round) and reported the first time it turns up
// under another one; t == 0 is skipped ("temp solution", :311-314).  The reference walks Go maps, so the ORDER of the
// reported ids is unspecified there; here it is responder order.  Host-side bookkeeping on ids (no crypto): a hash join.
int bftq_equivocation_scan_batch(const uint32_t* op_off, uint64_t n_ops, const uint8_t* status, const uint64_t* ts, const uint32_t* value_id,
                                 const uint32_t* signer_off, const uint64_t* signer_ids, uint32_t* out_off, uint64_t* out_ids, uint64_t cap_ids,
                                 uint64_t* n_ids) {
  if (!op_off || !out_off || !n_ids) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  const uint64_t n_items = n_ops ? op_off[n_ops] : 0;
  if (n_items && (!status || !ts || !value_id || !signer_off)) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  uint64_t total = 0;
  std::map<std::pair<uint64_t, uint64_t>, uint32_t> first_value;         // (t, signer) -> value id it was first seen with
  std::vector<uint64_t> revoked;
  for (uint64_t i = 0; i < n_ops; i++) {
    out_off[i] = (uint32_t)total;
    first_value.clear();
    revoked.clear();
    for (uint32_t p = op_off[i]; p < op_off[i + 1]; p++) {
      if (status[p] != 0 || ts[p] == 0) continue;
      for (uint32_t k = signer_off[p]; k < signer_off[p + 1]; k++) {
        const uint64_t id = signer_ids[k];
        auto key = std::make_pair(ts[p], id);
        auto it = first_value.find(key);
        if (it == first_value.end()) { first_value[key] = value_id[p]; continue; }
        if (it->second == value_id[p]) continue;
        bool seen = false;
        for (uint64_t r : revoked) if (r == id) { seen = true; break; }
        if (seen) continue;
        revoked.push_back(id);
        if (out_ids && total < cap_ids) out_ids[total] = id;
        total++;
      }
    }
  }
  out_off[n_ops] = (uint32_t)total;
  *n_ids = total;
  return BFTQ_OK;
}

int bftq_stats(bftq_engine* e, bftq_stats_t* out) {
  if (!e || !out) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  const EngineStats& s = e->stats;
  *out = bftq_stats_t{};
  out->items = s.items; out->launches = s.launches; out->h2d_bytes = s.h2d_bytes; out->d2h_bytes = s.d2h_bytes;
  out->packer_chunks = s.packer_chunks; out->packer_parse_ns = s.packer_parse_ns; out->packer_stage_ns = s.packer_stage_ns;
  out->packer_wait_ns = s.packer_wait_ns; out->msg_gpu_items = s.msg_gpu_items; out->msg_host_items = s.msg_host_items;
  out->unsupported_items = s.unsupported_items;
  out->numa_node = e->numa_node;
  out->numa_cpus = e->numa_valid ? (uint32_t)CPU_COUNT(&e->numa_cpus) : 0u;
  return BFTQ_OK;
}

int bftq_measure_int_peak(bftq_engine* e, double* macs_per_second) {
  if (!e || !macs_per_second) return fail(BFTQ_ERR_INVALID_ARG, "NULL argument");
  CU(cudaSetDevice(e->device));
  const int blocks = e->sm_count * 8, iters = 512 * kPeakUnroll;
  uint32_t* d = nullptr;
  CU(cudaMalloc((void**)&d, (size_t)blocks * 256 * 4));
  cudaEvent_t e0, e1;
  CU(cudaEventCreate(&e0));
  CU(cudaEventCreate(&e1));
  for (int w = 0; w < 20; w++) int_peak_kernel<<<blocks, 256>>>(d, 1234u + w, iters);   // warm clocks
  CU(cudaDeviceSynchronize());
  double best = 0;
  for (int rep = 0; rep < 5; rep++) {
    CU(cudaEventRecord(e0));
    for (int i = 0; i < 4; i++) int_peak_kernel<<<blocks, 256>>>(d, 99u + i, iters);
    CU(cudaEventRecord(e1));
    CU(cudaEventSynchronize(e1));
    float ms = 0;
    CU(cudaEventElapsedTime(&ms, e0, e1));
    double rate = 4.0 * blocks * 256.0 * iters * kPeakMacsPerIter / (ms * 1e-3);
    best = std::max(best, rate);
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(d);
  e->stats.launches += 40;                     // launched raw above: a check per launch would sit inside the timed window
  *macs_per_second = best;
  return BFTQ_OK;
}

}  // extern "C"
