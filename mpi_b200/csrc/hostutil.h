// hostutil.h -- host-only helpers of libb200mpi (no CUDA in this file, so they are unit-tested and
// run under ThreadSanitizer on a CPU box: tests/cpp/hostutil_test.cpp).
#pragma once
#include <errno.h>
#include <sched.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

namespace b200 {

// ---------------------------------------------------------------------------------------------
// NUMA placement.  The DMA engines of GPU g read and write host memory fastest on the socket the
// GPU hangs off (GPU0-3 / GPU4-7 of an HGX box sit on different sockets); rank processes started
// by torchrun / gompirun float across both.  Pinned buffers the library allocates and the helper
// threads that fill them are therefore placed on the GPU's node.
// ---------------------------------------------------------------------------------------------
static inline int read_int_file(const std::string& path, int dflt) {
  FILE* f = fopen(path.c_str(), "r");
  if (!f) return dflt;
  int v = dflt;
  if (fscanf(f, "%d", &v) != 1) v = dflt;
  fclose(f);
  return v;
}
// cpulist ("0-31,64-95") of a node -> cpu set; false when unknown
static inline bool cpus_of_node(int node, cpu_set_t& set) {
  CPU_ZERO(&set);
  if (node < 0) return false;
  FILE* f = fopen(("/sys/devices/system/node/node" + std::to_string(node) + "/cpulist").c_str(), "r");
  if (!f) return false;
  char buf[4096] = {0};
  const bool ok = fgets(buf, sizeof buf, f) != nullptr;
  fclose(f);
  if (!ok) return false;
  int count = 0;
  for (char* p = buf; *p;) {
    char* e;
    long a = strtol(p, &e, 10);
    if (e == p) break;
    long b = a;
    if (*e == '-') { p = e + 1; b = strtol(p, &e, 10); }
    for (long c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET((int)c, &set); ++count; }
    p = (*e == ',') ? e + 1 : e;
    if (*e != ',') break;
  }
  return count > 0;
}
// Runs fn with the calling thread's memory policy preferring `node` and its affinity on the node's
// CPUs (driver-side page allocation follows the calling thread), then restores both.
template <typename F>
static auto on_numa_node(int node, F fn) -> decltype(fn()) {
  cpu_set_t want, old;
  const bool have = cpus_of_node(node, want) && sched_getaffinity(0, sizeof old, &old) == 0;
  unsigned long mask[16] = {0}, old_mask[16] = {0};
  int old_mode = 0;
  bool have_policy = false;
  if (have) {
    have_policy = syscall(SYS_get_mempolicy, &old_mode, old_mask, sizeof old_mask * 8, nullptr, 0) == 0;
    if (node < (int)(sizeof mask * 8)) mask[node / (8 * sizeof(long))] |= 1ul << (node % (8 * sizeof(long)));
    syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, mask, sizeof mask * 8);
    // only narrow the affinity: a caller pinned elsewhere (taskset, cgroup cpuset) stays where it is
    cpu_set_t both;
    CPU_AND(&both, &want, &old);
    if (CPU_COUNT(&both) > 0) sched_setaffinity(0, sizeof both, &both);
  }
  auto r = fn();
  if (have) {
    // back to what the caller had (MPOL_DEFAULT when it could not be read)
    if (have_policy && old_mode != 0) syscall(SYS_set_mempolicy, old_mode, old_mask, sizeof old_mask * 8);
    else syscall(SYS_set_mempolicy, 0 /* MPOL_DEFAULT */, nullptr, 0);
    sched_setaffinity(0, sizeof old, &old);
  }
  return r;
}

// Helper threads that move bytes between a caller's pageable buffers and pinned bounce chunks.
// This is staging for the DMA engines, not a data path between ranks: every byte still travels
// host -> GPU -> NVLink -> GPU -> host.
struct CopyPool {
  struct Task { char* dst; const char* src; size_t n; std::atomic<int>* pending; };
  std::vector<std::thread> threads;
  std::mutex mu;
  std::condition_variable cv;
  std::deque<Task> q;
  bool stop = false;
  int nthreads = 0;
  bool running() const { return !threads.empty(); }
  void start(int n, int numa_node) {
    nthreads = std::max(n, 1);
    for (int i = 0; i < nthreads; ++i)
      threads.emplace_back([this, numa_node] {
        cpu_set_t set;
        if (cpus_of_node(numa_node, set)) sched_setaffinity(0, sizeof set, &set);
        for (;;) {
          Task t;
          {
            std::unique_lock<std::mutex> l(mu);
            cv.wait(l, [this] { return stop || !q.empty(); });
            if (q.empty()) return;
            t = q.front();
            q.pop_front();
          }
          memcpy(t.dst, t.src, t.n);
          t.pending->fetch_sub(1, std::memory_order_release);
        }
      });
  }
  void submit(char* dst, const char* src, size_t n, std::atomic<int>& pending) {
    if (n == 0) return;
    const size_t piece = std::max<size_t>(256u << 10, ((n + nthreads) / (nthreads + 1) + 4095) / 4096 * 4096);
    std::lock_guard<std::mutex> l(mu);
    for (size_t o = 0; o < n; o += piece) {
      pending.fetch_add(1, std::memory_order_relaxed);
      q.push_back({dst + o, src + o, std::min(piece, n - o), &pending});
    }
    cv.notify_all();
  }
  bool help_one() {
    Task t;
    {
      std::lock_guard<std::mutex> l(mu);
      if (q.empty()) return false;
      t = q.front();
      q.pop_front();
    }
    memcpy(t.dst, t.src, t.n);
    t.pending->fetch_sub(1, std::memory_order_release);
    return true;
  }
  void wait(std::atomic<int>& pending) { // the caller copies too while it waits
    while (pending.load(std::memory_order_acquire) > 0)
      if (!help_one()) sched_yield();
  }
  void shutdown() {
    {
      std::lock_guard<std::mutex> l(mu);
      stop = true;
    }
    cv.notify_all();
    for (auto& t : threads) t.join();
    threads.clear();
  }
};

// Elements per chunk of a pipelined host-slice collective (b200mpi.cu: host_pipeline): a multiple of
// 4096, at least 4096.  rows is n for Allgather (each chunk moves n rows), else 1.  In a multi-rank
// world every chunk launch pairs with the launch of the same number on every peer, so the chunk may
// only depend on what all ranks share: the knobs, the element size and n.  Whether this rank's
// buffer is pinned, registered or bounced is its own business, and the smaller of the two knobs
// serves all of them.  A world of one pairs nothing: a buffer that needs no bounce keeps the larger
// pipe chunk there.
static inline size_t pipe_chunk_elems(size_t es, size_t rows, int n, bool bounce, size_t pipe_chunk_bytes, size_t bounce_chunk_bytes) {
  const size_t bytes = n > 1 || bounce ? std::min(pipe_chunk_bytes, bounce_chunk_bytes) : pipe_chunk_bytes;
  return std::max<size_t>(bytes / rows / es, 4096) / 4096 * 4096;
}

// ---------------------------------------------------------------------------------------------
// Counter settings read at Init.
//   B200MPI_SCRUB_EVERY   launches between two flag scrubs: a power of two (rounded down, at least 2),
//                         clamped to max_scrub.  It can only lower the period: a longer one would let a
//                         flag word fall 2^31 behind and look "ahead".
//   B200MPI_EPOCH_START   (test hook) epoch of the first launch; must be 1 mod `stride`, the only values
//                         the launch schedule produces.
//   B200MPI_LL_SEQ_START  (test hook) the LL sequence number held after Init.
// Values are decimal.  A null string leaves the default.  Returns "" or what is wrong (Init then fails with B200MPI_ERR_ARG).
// ---------------------------------------------------------------------------------------------
struct CounterEnv {
  uint32_t scrub_every;
  uint32_t epoch_start = 1;
  uint32_t ll_seq_start = 0;
  bool preset = false; // B200MPI_EPOCH_START was given: preset the control region for that epoch
};
// Plain decimal digits only (no sign, blanks or base prefixes), at most 2^32 - 1.
static inline bool parse_u32(const char* s, uint32_t& v) {
  if (!s || !*s) return false;
  uint64_t x = 0;
  for (const char* p = s; *p; ++p) {
    if (*p < '0' || *p > '9') return false;
    x = x * 10 + (uint64_t)(*p - '0');
    if (x > 0xffffffffull) return false;
  }
  v = (uint32_t)x;
  return true;
}
static inline std::string parse_counter_env(const char* scrub, const char* epoch, const char* ll_seq, uint32_t max_scrub,
                                            uint32_t stride, CounterEnv& out) {
  out = CounterEnv();
  out.scrub_every = max_scrub;
  uint32_t v = 0;
  if (scrub) {
    if (!parse_u32(scrub, v)) return std::string("B200MPI_SCRUB_EVERY is not a decimal integer: '") + scrub + "'";
    uint32_t p2 = 2;
    while (p2 < max_scrub && p2 * 2 <= v) p2 *= 2;
    out.scrub_every = std::min(p2, max_scrub);
  }
  if (epoch) {
    if (!parse_u32(epoch, v)) return std::string("B200MPI_EPOCH_START is not a 32-bit decimal integer: '") + epoch + "'";
    if (v % stride != 1) return "B200MPI_EPOCH_START must be 1 mod " + std::to_string(stride) + ", got " + std::to_string(v);
    out.epoch_start = v;
    out.preset = true;
  }
  if (ll_seq) {
    if (!parse_u32(ll_seq, v)) return std::string("B200MPI_LL_SEQ_START is not a 32-bit decimal integer: '") + ll_seq + "'";
    out.ll_seq_start = v;
  }
  return "";
}

} // namespace b200
