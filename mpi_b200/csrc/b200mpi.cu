// b200mpi.cu -- host side of libb200mpi.so: the C ABI of include/b200mpi.h.
//
// What it replaces in the reference (/root/reference):
//   Network.Init / Finalize / Rank / Size   network.go:41-65,354-369   -> b200mpi_init & co.
//   Network.Send / Receive (+tagManager)    network.go:449-625         -> b200mpi_send / _recv
//   local (same-rank rendezvous)            network.go:388-446         -> same mailbox, own pair
//   AllReduce stub                          mpi.go:130                 -> b200mpi_allreduce, _bcast, _allgather
// The data never touches a socket: payloads move by sm_90a kernels (kernels.cuh) through the
// peer-mapped heaps (heap.h).  There is no CPU implementation of any data call: without a CUDA
// device every one of them fails with B200MPI_ERR_NO_DEVICE.
#include <cuda.h>
#include <cuda_runtime.h>
#include <ctype.h>
#include <errno.h>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <unistd.h>

#include <sys/syscall.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <limits>
#include <map>
#include <mutex>
#include <thread>
#include <set>
#include <string>
#include <variant>
#include <vector>

#include "../../include/b200mpi.h"
#include "ctrl.h"
#include "heap.h"
#include "hostutil.h"
#include "kernels.cuh"

namespace b200 {

// ---------------------------------------------------------------------------------------------
// mailbox: host shared memory (memfd) used for Send/Receive rendezvous, the role of the
// reference's tagManager + per-connection channels (network.go:449-497) and of `local`
// (network.go:388-446).  Control only: payload bytes never pass through it.
// ---------------------------------------------------------------------------------------------
constexpr int kSlotsPerPair = 16;
constexpr int kMsgRegions = 4;
enum SlotState : uint32_t { kFree = 0, kClaimed = 1, kPosted = 2, kMatched = 3, kDone = 4 };

struct alignas(128) MsgSlot {
  std::atomic<uint32_t> state;
  int32_t tag;
  uint32_t dtype;
  int32_t result;          // receiver's verdict, informational
  uint64_t count;          // elements
  uint64_t total_bytes;
  uint64_t chunk_bytes;    // size of one posted region (== total_bytes for a direct post)
  uint32_t nregions;       // ring of staging regions the chunks cycle through (1 for a direct post)
  uint32_t pad_;
  uint64_t region_off[kMsgRegions]; // offsets in the SENDER's heap
  std::atomic<uint64_t> posted; // bytes made available so far
  std::atomic<uint64_t> done;   // bytes consumed so far
};

struct Mailbox {
  MsgSlot slots[B200MPI_MAX_RANKS][B200MPI_MAX_RANKS][kSlotsPerPair]; // [src][dst][k]
};

struct TagSet { // duplicate in-flight {peer,tag} detection: tagManager.Register, network.go:464-472
  std::mutex mu;
  std::set<int> tags;
  bool add(int t) {
    std::lock_guard<std::mutex> g(mu);
    return tags.insert(t).second;
  }
  void remove(int t) {
    std::lock_guard<std::mutex> g(mu);
    tags.erase(t);
  }
};

// NUMA node of a GPU (sysfs entry of its PCI device); -1 unknown.
static int numa_node_of_gpu(int dev) {
  char id[32] = {0};
  if (cudaDeviceGetPCIBusId(id, sizeof id, dev) != cudaSuccess) { (void)cudaGetLastError(); return -1; }
  for (char* p = id; *p; ++p) *p = (char)tolower(*p);
  return read_int_file(std::string("/sys/bus/pci/devices/") + id + "/numa_node", -1);
}
struct Ctx {
  Ctrl ctrl;
  Driver drv;
  Heap heap;
  bool initialised = false;
  bool control_only = false;
  int dev = -1;
  int sm_count = 0;
  bool shared_device = false; // several ranks on one GPU (functional-test mode)
  Comm comm = {};
  uint32_t epoch = 1;
  uint32_t scrub_every = kScrubEvery; // power of two; B200MPI_SCRUB_EVERY lowers it so that a test can reach the scrub
  uint32_t* status_host = nullptr; // mapped pinned
  uint32_t* status_dev = nullptr;
  cudaStream_t own_stream = nullptr, stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaStream_t h2d_stream = nullptr, d2h_stream = nullptr; // host-slice pipeline
  std::vector<cudaEvent_t> pipe_events;
  size_t pipe_min_bytes = 8u << 20, pipe_chunk_bytes = 16u << 20;
  Mailbox* box = nullptr;
  TagSet sendtags[B200MPI_MAX_RANKS], recvtags[B200MPI_MAX_RANKS];
  std::mutex stream_mu;
  std::vector<cudaStream_t> stream_pool;
  int algo[4] = {0, 0, 0, 0};
  int max_blocks = 0;
  int64_t watchdog_ns = 120ll * 1000000000ll;
  size_t stage_chunk = 32u << 20;
  // staging for collectives on non-heap buffers: [0] send side, [1] recv side
  size_t stage_off[2] = {0, 0}, stage_len[2] = {0, 0};
  std::atomic<int64_t> launches{0};
  static constexpr int kBounceSlots = 4;
  char* bounce = nullptr;      // pinned ring for pageable host slices: [in kBounceSlots][out kBounceSlots] x bounce_chunk
  size_t bounce_chunk = 0, bounce_chunk_bytes = 4u << 20;
  int host_threads = 8;        // helper threads copying between pageable memory and the bounce ring
  CopyPool pool;
  // Host-slice Send/Receive up to kP2PBounceBytes: device-mapped pinned bounce buffers, one copy kernel
  // that reads / writes host memory itself, and a completion word the host spins on (no cudaMemcpy
  // staging by the driver, no stream synchronisation).
  static constexpr int kP2PBounces = 4;
  static constexpr size_t kP2PBounceBytes = 4u << 20;
  struct P2PBounce { char* host = nullptr; char* dev = nullptr; uint32_t seq = 0; bool busy = false; };
  P2PBounce p2p_bounce[kP2PBounces];
  std::mutex p2p_mu;
  bool p2p_fast = true;
  // Opt-in (B200MPI_HOST_REGISTER=1 / "host_register"): pin the caller's pageable buffers in place
  // (cudaHostRegister, cached by address range) instead of bouncing them.  Only for callers whose
  // buffers stay mapped for the life of the cache (a freed and re-mapped range would alias stale
  // pinned pages); off by default.
  bool host_register = false;
  std::vector<std::pair<uintptr_t, size_t>> registered; // LRU, most recent last
  int gpu_numa_node = -1;      // NUMA node of the bound GPU (-1 unknown): host buffers and helper threads go there
  size_t oneshot_max_bytes = 256u << 10;
  // Above a few MiB Bcast and Allgather stay on the P2P kernels, and the hybrid allreduce stays off,
  // until multicast delivery has been measured against plain P2P stores on H100.
  int hybrid_p2p_permille = 0; // Allreduce HYBRID: share of the message that goes the P2P way, in 1/1000
  int hybrid_p2p_blocks = 0;   // CTAs given to the P2P part (0 = sm_count - nvls_max_blocks)
  bool bcast_nvls2 = true;     // Bcast NVLS: scatter + multicast (1) or root-only multicast (0)
  size_t bcast_nvls_min = SIZE_MAX, allgather_nvls_min = SIZE_MAX; // AUTO thresholds (bytes)
  bool twoshot_unroll = true; // 0: 1/2/4 vectors per thread for n = 8/4/2, 1: 2/4/8
  int nvls_unroll = 2;      // multi-GPU switch tuning: not yet measured on H100 (tools/sweep.py re-derives it)
  int nvls_max_blocks = 48; // fewer requests in flight suit the switch reduction; not yet measured on H100
  size_t ll_max_bytes = 0; // AUTO uses the barrier-free LL allreduce for messages up to this size (<= 256 KiB)
  uint32_t ll_seq = 0;          // the last LL sequence number issued (ll_seq_next, kernels.cuh)
  bool ll_wrap_pending = false; // a resync crossed 2^32: the next LL call clears the lanes first
  // pinned, device-mapped bounce buffers: a small host-slice Allreduce is a memcpy + ONE kernel that
  // reads its input over PCIe and writes result + completion word to host memory
  char* ll_host = nullptr; char* ll_dev = nullptr; // [in kLLCells*8][out kLLCells*8][done word]
  size_t hybrid_min_bytes = 32u << 20;
  int nvls_min_ranks = 4; // below this the fused two-shot moves fewer bytes per link than NVLS
  size_t own_block_bytes = 1u << 20; // interleave granularity of slice ownership (Owner in kernels.cuh)
  // One-sided windows (b200mpi_win_create), indexed by window id: ids are handed out in call order and
  // never reused, so a freed window keeps its entry with live == false.  Every rank's heap offset and
  // size of each window, learnt at creation.  Dropped with the Ctx at teardown.
  struct Win {
    bool live;
    uint64_t off[B200MPI_MAX_RANKS], bytes[B200MPI_MAX_RANKS];
    uint32_t lock_cell;                    // its lock word in every rank's control region (kWinLockOff)
    uint8_t held[B200MPI_MAX_RANKS];       // the lock this rank holds on each target's window: 0 none, or a b200mpi_lock_type
    bool exposed, accessing;               // an exposure (win_post) / access (win_start) epoch of this rank is open
    uint8_t expose_group, access_group;    // the members of the open epochs, as rank masks
    uint16_t exposures[B200MPI_MAX_RANKS]; // exposure epochs this rank opened to each origin, mod 2^16
    uint16_t accesses[B200MPI_MAX_RANKS];  // access epochs this rank started on each target, mod 2^16
  };
  std::vector<Win> wins;
  std::vector<bool> lock_cell_used;        // kWinLockCells entries, one per lock word; a freed window's cell is reused
  // Host-mapped pinned words (allocated on first use): [0] the value fetch_and_op and compare_and_swap
  // fetch, [1] win_lock_try_kernel's verdict, [2] pscw_poll_kernel's arrivals (one byte per thread).
  uint64_t* rma_host = nullptr;
  uint64_t* rma_dev = nullptr;
};

static_assert(kHeapReserved == kCtrlBytes, "heap.h and kernels.cuh disagree about the control region");
static Ctx* g = nullptr;
static std::mutex g_mu;
static thread_local std::string t_err;

static int fail(int code, const std::string& msg) {
  t_err = msg;
  return code;
}
#define CUDA_OK(call)                                                                   \
  do {                                                                                  \
    cudaError_t _e = (call);                                                            \
    if (_e != cudaSuccess) return fail(B200MPI_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e)); \
  } while (0)

// Pinned host memory on the NUMA node of this rank's GPU.
static int numa_host_alloc(size_t bytes, void** p) {
  const cudaError_t e = on_numa_node(g->gpu_numa_node, [&] { return cudaHostAlloc(p, bytes ? bytes : 1, cudaHostAllocDefault); });
  if (e != cudaSuccess) return fail(B200MPI_ERR_CUDA, std::string("cudaHostAlloc: ") + cudaGetErrorString(e));
  return 0;
}

static size_t esize(int dtype) {
  switch (dtype) {
    case B200MPI_U8: return 1;
    case B200MPI_I64: return 8;
    case B200MPI_F32: return 4;
    case B200MPI_F64: return 8;
  }
  return 0;
}

static int need_init() { return g && g->initialised ? 0 : fail(B200MPI_ERR_NOT_INIT, "mpi: Init has not been called"); }

static thread_local int t_bound_dev = -1;
static int need_data_plane() {
  if (int rc = need_init()) return rc;
  if (g->control_only) return fail(B200MPI_ERR_NO_DEVICE, "no CUDA device bound (control-plane-only init); there is no CPU data path");
  if (t_bound_dev != g->dev) { // the CUDA "current device" is per host thread; Send/Receive come from any goroutine/thread
    if (cudaSetDevice(g->dev) != cudaSuccess) return fail(B200MPI_ERR_CUDA, "cudaSetDevice failed on a caller thread");
    t_bound_dev = g->dev;
  }
  return 0;
}

using Clock = std::chrono::steady_clock;
struct Spinner { // host-side wait with watchdog
  Clock::time_point t0 = Clock::now();
  uint32_t it = 0;
  int64_t limit_ns;
  explicit Spinner(int64_t ns) : limit_ns(ns) {}
  bool expired() const { return limit_ns > 0 && std::chrono::duration_cast<std::chrono::nanoseconds>(Clock::now() - t0).count() > limit_ns; }
  bool step() { // false => timed out
    if (++it < 4096) {
#if defined(__x86_64__)
      __builtin_ia32_pause();
#endif
      return true;
    }
    if ((it & 63) == 0) {
      if (limit_ns > 0 && std::chrono::duration_cast<std::chrono::nanoseconds>(Clock::now() - t0).count() > limit_ns) return false;
    }
    sched_yield();
    return true;
  }
};

static cudaStream_t borrow_stream() {
  {
    std::lock_guard<std::mutex> l(g->stream_mu);
    if (!g->stream_pool.empty()) {
      cudaStream_t s = g->stream_pool.back();
      g->stream_pool.pop_back();
      return s;
    }
  }
  cudaStream_t s = nullptr;
  cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
  return s;
}
static void return_stream(cudaStream_t s) {
  std::lock_guard<std::mutex> l(g->stream_mu);
  g->stream_pool.push_back(s);
}

// The cross-rank barriers pair CTAs by blockIdx and need all of them resident at once: one CTA per
// SM (512 threads, __launch_bounds__(.,1)), so a grid never exceeds the SM count.
static int block_cap() {
  int cap = g->max_blocks > 0 ? std::min(g->max_blocks, g->sm_count) : g->sm_count;
  return std::min(cap, kMaxBlocks);
}

static int grid_for(size_t units_per_rank, int unroll) {
  size_t per_block = (size_t)kThreads * unroll;
  size_t want = (units_per_rank + per_block - 1) / per_block;
  int cap = block_cap();
  if (want < 1) want = 1;
  return (int)(want > (size_t)cap ? cap : want);
}

// Every launch advances the epoch by kEpochStride whatever the algorithm (kernels.cuh), so ranks
// that disagreed about one call still agree about the flag values of the next.  `sig` is what this
// rank thinks the call is (make_sig), checked by sync_start on every rank.
static Comm next_comm(uint64_t sig) {
  // Every kScrubEvery-th launch (the same one on every rank: epochs move in lockstep) is preceded by
  // scrub_kernel, which rewrites every slot row so that no flag word can fall 2^31 behind the epoch.
  if (g->ctrl.n > 1 && ((g->epoch / kEpochStride) & (g->scrub_every - 1)) == g->scrub_every - 1) {
    Comm s = g->comm;
    s.epoch = g->epoch;
    s.end_epoch = g->epoch + kEpochStride - 1;
    s.sig = mix64(0x5c2b0000ull ^ ((uint64_t)kMaxBlocks << 8 | 0x5u));
    g->epoch += kEpochStride;
    scrub_kernel<<<kMaxBlocks, 32, 0, g->stream>>>(s);
    (void)cudaGetLastError();
  }
  Comm c = g->comm;
  c.epoch = g->epoch;
  c.sig = sig;
  c.end_epoch = g->epoch + kEpochStride - 1;
  g->epoch += kEpochStride;
  return c;
}

// After a failed collective the ranks may have issued different numbers of launches (chunked host
// paths) or LL calls: agree on max(epoch), max(ll_seq) over the control plane before the next call.
// Every rank sees the failure of a mismatched call (sync_start compares all signatures on every
// rank), so every rank comes here.
static void resync_after_error(bool peers_alive) {
  if (g->ctrl.n == 1) return;
  struct { uint32_t epoch, ll_seq, ll_wrap_pending; } mine = {g->epoch, g->ll_seq, g->ll_wrap_pending ? 1u : 0u}, all[B200MPI_MAX_RANKS];
  std::string err;
  // A mismatched call ends on every rank, so everybody comes here and the exchange is prompt.  After
  // a watchdog expiry a peer may be gone or stuck: do not trade one hang for another.
  const int64_t wait_ns = peers_alive ? 30ll * 1000000000ll : 2ll * 1000000000ll;
  if (g->ctrl.allgather(&mine, sizeof mine, all, err, wait_ns) != 0) return; // nothing to agree with
  for (int r = 0; r < g->ctrl.n; ++r) {
    if (!flag_reached(g->epoch, all[r].epoch)) g->epoch = all[r].epoch;
    if (!flag_reached(g->ll_seq, all[r].ll_seq)) g->ll_seq = all[r].ll_seq;
    if (all[r].ll_wrap_pending) g->ll_wrap_pending = true;
  }
  g->epoch += kEpochStride;
  // keep the parity, skip cells a failed call may have half written; when this crosses 2^32 the next
  // LL call clears the lanes first
  const LLSeqNext next = ll_seq_next(g->ll_seq, 2);
  g->ll_seq = next.seq;
  if (next.wrapped) g->ll_wrap_pending = true;
}

static int check_status() {
  if (g->status_host && *(volatile uint32_t*)g->status_host) {
    const uint32_t st = *(volatile uint32_t*)g->status_host;
    *(volatile uint32_t*)g->status_host = 0;
    resync_after_error(st == 2u);
    if (st == 2u) return fail(B200MPI_ERR_PEER, "mismatched collective: ranks disagree on the call (collective, count, dtype, op, root, algorithm or grid); buffers were left untouched");
    return fail(B200MPI_ERR_TIMEOUT, "device-side watchdog: a peer did not reach the collective in time");
  }
  return 0;
}

// What this rank thinks the call is, folded into one word; equal on every rank of a well-formed
// call.  coll: 0 allreduce, 1 bcast, 2 allgather, 3 barrier, 4 reduce_scatter, 5 reduce, 6 alltoall,
// 7 gather(v), 8 scatter(v), 9 allgatherv (these three carry a hash of the counts table in `total`),
// 10 alltoallv (whose ranks hold different tables: each adds its table digest to the signature it
// announces, see sync_start_pairs in kernels.cuh), 11 scan, 12 exscan, 13 reduce_scatterv (which
// carries the table hash in `total`, as 7-9 do), 14 allreduce_loc and reduce_loc (extra = op |
// (root + 1) << 4, root -1 for allreduce_loc), 15 win_fence and win_free (count = the window id).
// `total` is the element count of the whole user call when the launch is one chunk of a pipelined
// host-slice call (ranks that disagree about the total then disagree from the first chunk on).
static uint64_t make_sig(int coll, int dtype, int extra, int algo, size_t count, size_t total = 0) {
  uint64_t h = mix64((uint64_t)count + 0x9e3779b97f4a7c15ull);
  h = mix64(h ^ ((uint64_t)(coll & 15) << 40 | (uint64_t)(dtype & 15) << 32 | (uint64_t)(extra & 0xffff) << 16 | (uint64_t)(algo & 0xffff)));
  return mix64(h ^ (uint64_t)total);
}
// The grid is part of the signature: the barriers pair CTAs by blockIdx.
static void sig_grid(Comm& c, int blocks) { c.sig = mix64(c.sig ^ ((uint64_t)blocks << 8 | 0x5u)); }

static int launch_check(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(B200MPI_ERR_CUDA, std::string(what) + " launch failed: " + cudaGetErrorString(e));
  g->launches.fetch_add(1, std::memory_order_relaxed);
  return 0;
}

// One collective launch: take the epoch, fold the grid into the signature, launch kernel(comm,
// args...) and check the launch.  Callers settle the algorithm and the grid first, so a launch that
// does not happen takes no epoch.
template <typename... P, typename... A>
static int launch_coll(void (*kernel)(Comm, P...), const char* what, uint64_t sig, int blocks, int threads, size_t smem, cudaStream_t s, A... args) {
  Comm c = next_comm(sig);
  sig_grid(c, blocks);
  kernel<<<blocks, threads, smem, s>>>(c, args...);
  return launch_check(what);
}

// The grid of launch_copy (and of accumulate_kernel) for `bytes`: one 256-thread CTA per 64 KiB, up
// to one CTA per SM (or max_blocks).
static int copy_grid(size_t bytes) {
  constexpr size_t kPerBlock = 256 * 16 * 16; // bytes one CTA of copy_bytes_kernel moves per grid pass
  const size_t want = (bytes + kPerBlock - 1) / kPerBlock;
  const size_t cap = g->max_blocks > 0 ? (size_t)g->max_blocks : (size_t)g->sm_count;
  return (int)std::max<size_t>(1, std::min(want, cap));
}

// dst <- src on `s` with the library's own copy kernel (local HBM or peer mapping), any alignment:
// 256 threads x 16 vectors in flight per thread, up to one CTA per SM (or max_blocks).
static int launch_copy(void* dst, const void* src, size_t bytes, cudaStream_t s) {
  if (bytes == 0) return 0;
  copy_bytes_kernel<16, 256, 1><<<copy_grid(bytes), 256, 0, s>>>((unsigned char*)dst, (const unsigned char*)src, bytes);
  return launch_check("copy_bytes_kernel");
}

// dst <- src where both ends are memory of this rank's GPU: copy_local_kernel with one thread per
// 16-byte vector when src and dst agree mod 16 and the copy is at least kLocalCopyMinBytes (a grid
// of up to 2^31 - 1 CTAs, or max_blocks), else launch_copy.  Below 8 MiB the grid-stride kernel was
// as fast or faster on an H100 SXM (400 W): at 4 MiB 4.5 us against 6.7-7.9 us per call.
static constexpr size_t kLocalCopyMinBytes = 8u << 20;
static int launch_local_copy(void* dst, const void* src, size_t bytes, cudaStream_t s) {
  if (bytes == 0) return 0;
  if ((((uintptr_t)dst ^ (uintptr_t)src) & 15) || bytes < kLocalCopyMinBytes) return launch_copy(dst, src, bytes, s);
  const size_t want = (bytes / 16 + kLocalCopyThreads - 1) / kLocalCopyThreads;
  const size_t cap = g->max_blocks > 0 ? (size_t)g->max_blocks : (size_t)INT32_MAX;
  const int blocks = (int)std::max<size_t>(1, std::min(want, cap));
  copy_local_kernel<<<blocks, kLocalCopyThreads, 0, s>>>((unsigned char*)dst, (const unsigned char*)src, bytes);
  return launch_check("copy_local_kernel");
}

// ---------------------------------------------------------------------------------------------
// kernel dispatch
// ---------------------------------------------------------------------------------------------
// log2 of the ownership block, in 16-byte vectors: at most own_block_bytes, at most the per-rank
// share (so every rank owns something), at least `min_shift`.  Function of (count, n) only.
static uint32_t own_shift(size_t nvec, int n, uint32_t min_shift) {
  size_t per = std::max<size_t>((nvec + n - 1) / n, 1);
  uint32_t sh = 0;
  while (((size_t)2 << sh) <= per) ++sh;                        // floor(log2(per))
  uint32_t cap = 0;
  while (((size_t)32 << cap) <= g->own_block_bytes) ++cap;      // floor(log2(own_block_bytes / 16))
  sh = std::min(sh, cap);
  return std::max(sh, min_shift);
}

template <int V> using ic = std::integral_constant<int, V>;

// The template arguments (NR, UNROLL) of the owner-computes kernels, the two-shot Allreduce at its
// default unroll and Scan, for a world of n ranks: f(NR, UNROLL) as integral constants.  NR = 0 is
// the instance for any n.  UNROLL is the largest per (n, element size) for which ptxas reports no
// spill: 8-byte min/max spilled at 8 vectors per thread.
template <typename T, typename F>
static int with_owner_tiling(int n, F&& f) {
  if (n == 2) return f(ic<2>{}, ic<sizeof(T) == 4 ? 8 : 4>{});
  if (n == 4) return f(ic<4>{}, ic<4>{});
  if (n == 8) return f(ic<8>{}, ic<2>{});
  return f(ic<0>{}, ic<1>{});
}

// only_dst: -1 allreduce, else the root of a Reduce (twoshot / nvls only)
template <typename T, typename Op>
static int launch_allreduce_body_t(int algo, uint64_t sig, uint64_t so, uint64_t ro, size_t count, int only_dst, cudaStream_t s) {
  const int n = g->ctrl.n;
  constexpr int EPV = 16 / sizeof(T);
  const size_t nvec = (count + EPV - 1) / EPV;
  const size_t per = (nvec + n - 1) / n;
  const uint32_t sh = own_shift(nvec, n, algo == B200MPI_ALGO_TWOSHOT_SMEM ? 8 : 0);
  switch (algo) {
    case B200MPI_ALGO_TWOSHOT: {
      auto go = [&](auto nr, auto unroll) {
        return launch_coll(allreduce_twoshot_kernel<T, Op, nr, unroll>, "allreduce_twoshot_kernel", sig, grid_for(per, unroll), kThreads, 0, s, so, ro, count, sh, only_dst);
      };
      if (g->twoshot_unroll) return with_owner_tiling<T>(n, go);
      if (n == 2) return go(ic<2>{}, ic<4>{});
      if (n == 4) return go(ic<4>{}, ic<2>{});
      if (n == 8) return go(ic<8>{}, ic<1>{});
      return go(ic<0>{}, ic<1>{});
    }
    case B200MPI_ALGO_RING:
      return launch_coll(allreduce_ring_kernel<T, Op>, "allreduce_ring_kernel", sig, grid_for(per, 4), kThreads, 0, s, so, ro, count);
    case B200MPI_ALGO_TWOSHOT_SMEM: {
      const size_t tiles = (per * 16 + kSmemChunk - 1) / kSmemChunk;
      const int blocks = (int)std::max<size_t>(1, std::min<size_t>(tiles, (size_t)block_cap()));
#define B200_SMEM(NRV)                                                                                           \
  {                                                                                                              \
    const size_t smem = (size_t)(kSmemStages * NRV + kSmemOutStages) * kSmemChunk;                               \
    static bool attr_set = false;                                                                                \
    if (!attr_set) {                                                                                             \
      cudaFuncSetAttribute(allreduce_twoshot_smem_kernel<T, Op, NRV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
      attr_set = true;                                                                                           \
    }                                                                                                            \
    return launch_coll(allreduce_twoshot_smem_kernel<T, Op, NRV>, "allreduce_twoshot_smem_kernel", sig, blocks, kSmemThreads, smem, s, so, ro, count, sh); \
  }
      if (n == 2) B200_SMEM(2)
      else if (n == 4) B200_SMEM(4)
      else B200_SMEM(8)
#undef B200_SMEM
    }
  }
  return fail(B200MPI_ERR_UNSUPPORTED, "allreduce: algorithm not available for this dtype/op");
}

// One-shot geometry, shared by pick (which must know whether the call fits) and launch: a function
// of (count, n, element size, grid cap) only.
struct OneshotPlan { bool shfl; int blocks; size_t rounds; };
static OneshotPlan oneshot_plan(size_t count, size_t es) {
  const int n = g->ctrl.n;
  const size_t epv = 16 / es;
  const size_t nvec = (count + epv - 1) / epv;
  OneshotPlan p;
  p.shfl = (n == 2 || n == 4 || n == 8) && nvec <= 4096;
  p.blocks = p.shfl ? grid_for(nvec * n, 1) : grid_for(nvec, 1);
  const size_t per_round = (size_t)p.blocks * kThreads;
  // one mid-barrier value per round (upper bound: the scalar rounds of the unaligned path)
  p.rounds = (count + per_round - 1) / per_round + (p.shfl ? (nvec * n + per_round - 1) / per_round : 0) + 2;
  return p;
}

template <typename T, typename Op>
static int launch_allreduce_t(int algo, uint64_t sig, uint64_t so, uint64_t ro, size_t count, cudaStream_t s) {
  const int n = g->ctrl.n;
  if (algo != B200MPI_ALGO_ONESHOT) return launch_allreduce_body_t<T, Op>(algo, sig, so, ro, count, -1, s);
  const OneshotPlan p = oneshot_plan(count, sizeof(T));
  if (p.rounds > kMaxMids) return fail(B200MPI_ERR_UNSUPPORTED, "allreduce: message too large for the one-shot algorithm");
  auto go = [&](auto kernel, const char* what) { return launch_coll(kernel, what, sig, p.blocks, kThreads, 0, s, so, ro, count); };
  if (p.shfl) {
    if (n == 2) return go(allreduce_oneshot_shfl_kernel<T, Op, 2>, "allreduce_oneshot_shfl_kernel");
    if (n == 4) return go(allreduce_oneshot_shfl_kernel<T, Op, 4>, "allreduce_oneshot_shfl_kernel");
    return go(allreduce_oneshot_shfl_kernel<T, Op, 8>, "allreduce_oneshot_shfl_kernel");
  }
  if (n == 2) return go(allreduce_oneshot_kernel<T, Op, 2>, "allreduce_oneshot_kernel");
  if (n == 4) return go(allreduce_oneshot_kernel<T, Op, 4>, "allreduce_oneshot_kernel");
  if (n == 8) return go(allreduce_oneshot_kernel<T, Op, 8>, "allreduce_oneshot_kernel");
  return go(allreduce_oneshot_kernel<T, Op, 0>, "allreduce_oneshot_kernel");
}

static int nvls_blocks(size_t per, int u) {
  int blocks = grid_for(per, u);
  if (g->max_blocks == 0 && blocks > g->nvls_max_blocks) blocks = g->nvls_max_blocks;
  return blocks;
}

template <typename T, typename Op>
static int launch_allreduce_nvls_t(uint64_t sig, uint64_t so, uint64_t ro, size_t count, int only_dst, cudaStream_t s) {
  const int n = g->ctrl.n;
  constexpr int EPV = 16 / sizeof(T);
  const size_t nvec = (count + EPV - 1) / EPV;
  const size_t per = (nvec + n - 1) / n;
  const uint32_t sh = own_shift(nvec, n, 0);
  int u = g->nvls_unroll;
  if (u != 1 && u != 2 && u != 8) u = 4;
  auto go = [&](auto kernel) { return launch_coll(kernel, "allreduce_nvls_kernel", sig, nvls_blocks(per, u), kThreads, 0, s, so, ro, count, sh, only_dst); };
  switch (u) {
    case 1: return go(allreduce_nvls_kernel<T, Op, 1>);
    case 2: return go(allreduce_nvls_kernel<T, Op, 2>);
    case 8: return go(allreduce_nvls_kernel<T, Op, 8>);
  }
  return go(allreduce_nvls_kernel<T, Op, 4>);
}

// NVLS for [0, split) + fused P2P two-shot for the rest, in one kernel (kernels.cuh).  The split is
// cut on ownership-block boundaries of both parts and depends on (count, n, parameters) only.
template <typename T, typename Op>
static int launch_allreduce_hybrid_t(uint64_t sig, uint64_t so, uint64_t ro, size_t count, cudaStream_t s) {
  const int n = g->ctrl.n;
  constexpr int EPV = 16 / sizeof(T);
  const size_t nvec = count / EPV; // whole vectors; the tail goes with the P2P part
  size_t p2p_vec = (size_t)((double)nvec * g->hybrid_p2p_permille / 1000.0);
  const size_t gran = (size_t)n << 8; // n blocks of 4 KiB: every rank owns the same share of both parts
  p2p_vec = p2p_vec / gran * gran;
  const size_t split = nvec - p2p_vec;
  if (n != 8 && n != 4 && n != 2) return fail(B200MPI_ERR_UNSUPPORTED, "allreduce: the hybrid algorithm needs 2, 4 or 8 ranks");
  if (split == 0 || p2p_vec == 0) return launch_allreduce_nvls_t<T, Op>(sig, so, ro, count, -1, s);
  const uint32_t sh_n = own_shift(split, n, 0), sh_p = own_shift(p2p_vec, n, 0);
  int u = g->nvls_unroll == 4 ? 4 : 2;
  const int nb_nvls = nvls_blocks((split + n - 1) / n, u);
  int nb_p2p = g->hybrid_p2p_blocks > 0 ? g->hybrid_p2p_blocks : block_cap() - nb_nvls;
  nb_p2p = std::max(1, std::min(nb_p2p, block_cap() - nb_nvls));
  if (nb_nvls + nb_p2p > block_cap()) return launch_allreduce_nvls_t<T, Op>(sig, so, ro, count, -1, s);
  auto go = [&](auto kernel) {
    return launch_coll(kernel, "allreduce_hybrid_kernel", sig, nb_nvls + nb_p2p, kThreads, 0, s, so, ro, count, sh_n, sh_p, split, (unsigned)nb_nvls);
  };
#define B200_HYB(NRV, UP) return u == 4 ? go(allreduce_hybrid_kernel<T, Op, NRV, 4, UP>) : go(allreduce_hybrid_kernel<T, Op, NRV, 2, UP>);
  if (n == 8) B200_HYB(8, 2)
  if (n == 4) B200_HYB(4, 4)
  B200_HYB(2, 4)
#undef B200_HYB
}

// The reductions the kernels are instantiated for: f32, f64 and i64 with sum, max and min.  Returns
// f(T{}, Op{}) for (dtype, op), or otherwise() for any other pair.
template <typename T, typename F, typename G>
static auto with_op(int op, F& f, G& otherwise) {
  switch (op) {
    case B200MPI_SUM: return f(T{}, OpSum{});
    case B200MPI_MAX: return f(T{}, OpMax{});
    case B200MPI_MIN: return f(T{}, OpMin{});
  }
  return otherwise();
}
template <typename F, typename G>
static auto with_reduction(int dtype, int op, F&& f, G&& otherwise) {
  switch (dtype) {
    case B200MPI_F32: return with_op<float>(op, f, otherwise);
    case B200MPI_F64: return with_op<double>(op, f, otherwise);
    case B200MPI_I64: return with_op<long long>(op, f, otherwise);
  }
  return otherwise();
}

// The reductions the switch performs in multimem.ld_reduce: sums of f32, f64 and i64, min/max of
// i64 only.  The NVLS kernels are instantiated for exactly these.
template <typename T, typename Op>
static constexpr bool switch_reduces() { return std::is_same<Op, OpSum>::value || std::is_same<T, long long>::value; }

static bool nvls_supports(int dtype, int op) {
  return with_reduction(dtype, op, [](auto t, auto o) { return switch_reduces<decltype(t), decltype(o)>(); }, [] { return false; });
}

// `total`: element count of the whole user call when this launch is one chunk of it, else 0.
static int launch_allreduce(int algo, int dtype, int op, uint64_t so, uint64_t ro, size_t count, cudaStream_t s, size_t total = 0) {
  const uint64_t sig = make_sig(0, dtype, op, algo, count, total);
  const bool nvls = algo == B200MPI_ALGO_NVLS || algo == B200MPI_ALGO_HYBRID;
  const char* nvls_only = "allreduce: NVLS supports sum (f32,f64,i64) and min/max (i64) only";
  return with_reduction(
      dtype, op,
      [&](auto t, auto o) {
        using T = decltype(t);
        using Op = decltype(o);
        if (!nvls) return launch_allreduce_t<T, Op>(algo, sig, so, ro, count, s);
        if constexpr (switch_reduces<T, Op>())
          return algo == B200MPI_ALGO_HYBRID ? launch_allreduce_hybrid_t<T, Op>(sig, so, ro, count, s) : launch_allreduce_nvls_t<T, Op>(sig, so, ro, count, -1, s);
        else return fail(B200MPI_ERR_UNSUPPORTED, nvls_only);
      },
      [&] { return fail(B200MPI_ERR_UNSUPPORTED, nvls ? nvls_only : "allreduce: unsupported dtype/op (need f32, f64 or i64 with sum/max/min)"); });
}

// Reduce to `root`: the owner-reduces bodies with a single destination.
static int launch_reduce(int algo, int dtype, int op, uint64_t so, uint64_t ro, size_t count, int root, cudaStream_t s) {
  const uint64_t sig = make_sig(5, dtype, op | (root << 4), algo, count);
  return with_reduction(
      dtype, op,
      [&](auto t, auto o) {
        using T = decltype(t);
        using Op = decltype(o);
        if (algo != B200MPI_ALGO_NVLS) return launch_allreduce_body_t<T, Op>(B200MPI_ALGO_TWOSHOT, sig, so, ro, count, root, s);
        if constexpr (switch_reduces<T, Op>()) return launch_allreduce_nvls_t<T, Op>(sig, so, ro, count, root, s);
        else return fail(B200MPI_ERR_UNSUPPORTED, "reduce: NVLS supports sum (f32,f64,i64) and min/max (i64) only");
      },
      [] { return fail(B200MPI_ERR_UNSUPPORTED, "reduce: unsupported dtype/op (need f32, f64 or i64 with sum/max/min)"); });
}

static int launch_reduce_scatter(int algo, int dtype, int op, uint64_t so, uint64_t ro, size_t count, cudaStream_t s) {
  const bool nvls = algo == B200MPI_ALGO_NVLS && op == B200MPI_SUM; // the switch form is instantiated for sums
  const uint64_t sig = make_sig(4, dtype, op, nvls ? B200MPI_ALGO_NVLS : B200MPI_ALGO_TWOSHOT, count);
  return with_reduction(
      dtype, op,
      [&](auto t, auto o) {
        using T = decltype(t);
        using Op = decltype(o);
        constexpr int EPV = 16 / sizeof(T);
        const size_t nvec = (count + EPV - 1) / EPV;
        if constexpr (std::is_same<Op, OpSum>::value)
          if (nvls) return launch_coll(reduce_scatter_nvls_kernel<T, OpSum, 2>, "reduce_scatter_nvls_kernel", sig, nvls_blocks(nvec, 2), kThreads, 0, s, so, ro, count);
        return launch_coll(reduce_scatter_kernel<T, Op, 2>, "reduce_scatter_kernel", sig, grid_for(nvec, 2), kThreads, 0, s, so, ro, count);
      },
      [&] {
        const bool known_dtype = dtype == B200MPI_F32 || dtype == B200MPI_F64 || dtype == B200MPI_I64;
        return known_dtype ? fail(B200MPI_ERR_ARG, "reduce_scatter: unknown op") : fail(B200MPI_ERR_UNSUPPORTED, "reduce_scatter: dtype must be f32, f64 or i64");
      });
}

// Scan / Exscan: one algorithm, the two-shot ownership, grid and (NR, UNROLL).
static int launch_scan(bool exclusive, int dtype, int op, uint64_t so, uint64_t ro, size_t count, cudaStream_t s) {
  const uint64_t sig = make_sig(exclusive ? 12 : 11, dtype, op, 0, count);
  return with_reduction(
      dtype, op,
      [&](auto t, auto o) {
        using T = decltype(t);
        using Op = decltype(o);
        const int n = g->ctrl.n;
        constexpr int EPV = 16 / sizeof(T);
        const size_t nvec = (count + EPV - 1) / EPV;
        const size_t per = (nvec + n - 1) / n;
        const uint32_t sh = own_shift(nvec, n, 0);
        auto go = [&](auto kernel, int unroll) { return launch_coll(kernel, "scan_kernel", sig, grid_for(per, unroll), kThreads, 0, s, so, ro, count, sh); };
        return with_owner_tiling<T>(n, [&](auto nr, auto unroll) {
          return exclusive ? go(scan_kernel<T, Op, nr, unroll, true>, unroll) : go(scan_kernel<T, Op, nr, unroll, false>, unroll);
        });
      },
      [&] { return fail(B200MPI_ERR_UNSUPPORTED, "scan: unsupported dtype/op (need f32, f64 or i64 with sum/max/min)"); });
}

// The value-location reductions the two-shot body is instantiated for: {f32, f64, i64} pairs with
// MAXLOC (op MAX) and MINLOC (op MIN).  Returns f(Loc<V>{}, Op{}), or otherwise() for any other pair.
template <typename F, typename G>
static auto with_loc_reduction(int dtype, int op, F&& f, G&& otherwise) {
  auto by_op = [&](auto v) {
    using P = Loc<decltype(v)>;
    switch (op) {
      case B200MPI_MAX: return f(P{}, OpMaxLoc{});
      case B200MPI_MIN: return f(P{}, OpMinLoc{});
    }
    return otherwise();
  };
  switch (dtype) {
    case B200MPI_F32: return by_op(float{});
    case B200MPI_F64: return by_op(double{});
    case B200MPI_I64: return by_op((long long)0);
  }
  return otherwise();
}

// AllreduceLoc (root < 0) and ReduceLoc: one algorithm, the two-shot Allreduce kernel over 16-byte
// pairs (one pair per vector) with its grid and (NR, UNROLL).  Signature code 14 carries op, root + 1,
// dtype and count, so a rank calling Allreduce, the other of the two, or another op, dtype, count or
// root ends the call as B200MPI_ERR_PEER on every rank.
static int launch_allreduce_loc(int dtype, int op, uint64_t so, uint64_t ro, size_t count, int root, cudaStream_t s) {
  const uint64_t sig = make_sig(14, dtype, op | (root + 1) << 4, 0, count);
  return with_loc_reduction(
      dtype, op,
      [&](auto t, auto o) {
        using T = decltype(t);
        using Op = decltype(o);
        const int n = g->ctrl.n;
        const size_t per = (count + n - 1) / n;
        const uint32_t sh = own_shift(count, n, 0);
        return with_owner_tiling<T>(n, [&](auto nr, auto unroll) {
          return launch_coll(allreduce_twoshot_kernel<T, Op, nr, unroll>, "allreduce_twoshot_kernel", sig, grid_for(per, unroll), kThreads, 0, s, so, ro, count, sh, root);
        });
      },
      [] { return fail(B200MPI_ERR_UNSUPPORTED, "allreduce_loc: unsupported dtype/op (need f32, f64 or i64 pairs with max/min)"); });
}

// AUTO for Allreduce: best busbw / latency per (n, size) among the variants.  The multi-GPU thresholds
// have not been measured on H100 yet (tools/sweep.py re-derives them on a box with 2/4/8 GPUs).
// chunk: the launch is one piece of a pipelined host-slice call, where the barrier-free LL kernel
// (own sequence numbers, no heap offsets) does not apply.
static int pick_allreduce(size_t bytes, int dtype, int op, bool chunk = false) {
  const int n = g->ctrl.n;
  const bool pow2 = n == 2 || n == 4 || n == 8;
  const size_t es = esize(dtype);
  int forced = g->algo[B200MPI_COLL_ALLREDUCE];
  const bool can_nvls = g->heap.mc_base && nvls_supports(dtype, op);
  if (forced == B200MPI_ALGO_TWOSHOT_SMEM && !pow2) forced = B200MPI_ALGO_TWOSHOT;
  if (forced == B200MPI_ALGO_NVLS && !can_nvls) forced = 0;
  if (forced == B200MPI_ALGO_HYBRID && !(can_nvls && pow2 && g->hybrid_p2p_permille > 0)) forced = can_nvls ? B200MPI_ALGO_NVLS : 0;
  if (forced == B200MPI_ALGO_LL && (bytes > ll_cells(g->ctrl.n) * 8 || chunk)) forced = chunk ? B200MPI_ALGO_ONESHOT : 0;
  if (forced == B200MPI_ALGO_ONESHOT && es && oneshot_plan(bytes / es, es).rounds > kMaxMids) forced = B200MPI_ALGO_TWOSHOT;
  if (forced) return forced;
  if (g->ll_max_bytes && bytes <= g->ll_max_bytes && !chunk) return B200MPI_ALGO_LL;
  const bool nvls = can_nvls && n >= g->nvls_min_ranks;
  const int big = pow2 ? B200MPI_ALGO_TWOSHOT_SMEM : B200MPI_ALGO_TWOSHOT;
  if (n >= 8) {
    if (nvls) return (pow2 && g->hybrid_p2p_permille > 0 && bytes >= g->hybrid_min_bytes) ? B200MPI_ALGO_HYBRID : B200MPI_ALGO_NVLS;
    return bytes < (2u << 20) ? B200MPI_ALGO_TWOSHOT : big;
  }
  if (n >= 3) {
    if (nvls && bytes <= (4u << 20)) return B200MPI_ALGO_NVLS;
    if (!nvls && bytes <= g->oneshot_max_bytes) return B200MPI_ALGO_ONESHOT;
    return bytes < (2u << 20) ? B200MPI_ALGO_TWOSHOT : big;
  }
  if (bytes <= g->oneshot_max_bytes) return B200MPI_ALGO_ONESHOT;
  return B200MPI_ALGO_TWOSHOT; // n == 2: the LDG and the TMA-staged two-shot move the same bytes per link
}

// AUTO for Bcast: the switch multicast wins up to a few MiB (one store stream, no second hop); the
// scatter + multicast form keeps winning above that (every byte leaves root once, every ingress
// link fills at the same time); without NVLS the fused pull-slice + push.
static int pick_bcast(size_t bytes) {
  const int n = g->ctrl.n;
  int forced = g->algo[B200MPI_COLL_BCAST];
  if (forced == B200MPI_ALGO_NVLS && !g->heap.mc_base) forced = 0;
  if (forced == B200MPI_ALGO_RING || forced == B200MPI_ALGO_TWOSHOT_SMEM || forced == B200MPI_ALGO_HYBRID || forced == B200MPI_ALGO_LL) forced = B200MPI_ALGO_TWOSHOT;
  if (forced) return forced;
  if (g->heap.mc_base && bytes % 16 == 0 && n >= 3 && (bytes <= (4u << 20) || (g->bcast_nvls2 && bytes >= g->bcast_nvls_min))) return B200MPI_ALGO_NVLS;
  if (n == 2 || bytes <= (64u << 10)) return B200MPI_ALGO_ONESHOT;
  return B200MPI_ALGO_TWOSHOT;
}

static int pick_allgather(size_t bytes_per_rank) {
  int forced = g->algo[B200MPI_COLL_ALLGATHER];
  if (forced == B200MPI_ALGO_RING) return forced;
  if (forced == B200MPI_ALGO_NVLS && g->heap.mc_base) return forced;
  if (forced) return B200MPI_ALGO_ONESHOT;
  if (g->heap.mc_base && g->ctrl.n >= 3 && bytes_per_rank % 16 == 0 && bytes_per_rank >= g->allgather_nvls_min) return B200MPI_ALGO_NVLS;
  return B200MPI_ALGO_ONESHOT; // direct push
}

static int pick_reduce_scatter(size_t, int dtype, int op) {
  int forced = g->algo[B200MPI_COLL_REDUCE_SCATTER];
  const bool can = g->heap.mc_base && op == B200MPI_SUM && nvls_supports(dtype, op);
  if (forced == B200MPI_ALGO_NVLS) return can ? B200MPI_ALGO_NVLS : B200MPI_ALGO_TWOSHOT;
  if (forced) return B200MPI_ALGO_TWOSHOT;
  return can && g->ctrl.n >= g->nvls_min_ranks ? B200MPI_ALGO_NVLS : B200MPI_ALGO_TWOSHOT;
}

// Returns f(U{}) for the widest access unit U (uint4, 8, 4 or 1 byte) dividing m, the OR of THIS
// rank's offsets, sizes and displacements.  Peers may be aligned differently: after the start
// barrier every rank knows all offsets and drops to the byte-wide body if some peer's are narrower
// than its own unit (kernels.cuh: all_aligned_to).  Ranks may so instantiate different units but
// must launch the same number of CTAs, because the barriers pair CTAs by blockIdx: a grid never
// depends on U.
template <typename F>
static int with_unit(uint64_t m, F&& f) {
  if ((m & 15) == 0) return f(uint4{});
  if ((m & 7) == 0) return f(0ull);
  if ((m & 3) == 0) return f(0u);
  return f((unsigned char)0);
}

// Bcast of `bytes` at heap offset `off` on every... (each rank passes its own offset)
static int launch_bcast(int algo, int dtype, size_t count, uint64_t off, size_t bytes, int root, cudaStream_t s, size_t total = 0) {
  const uint64_t sig = make_sig(1, dtype, root, algo, count, total);
  const int n = g->ctrl.n;
  const size_t nvec = bytes / 16 + 1;
  if (algo == B200MPI_ALGO_NVLS) {
    if (g->bcast_nvls2)
      return launch_coll(bcast_nvls2_kernel<4>, "bcast_nvls2_kernel", sig, grid_for((nvec + n - 1) / n, 4), kThreads, 0, s, off, bytes, root, own_shift(nvec, n, 0));
    return launch_coll(bcast_nvls_kernel<4>, "bcast_nvls_kernel", sig, grid_for(nvec, 4), kThreads, 0, s, off, bytes, root);
  }
  const int mode = algo == B200MPI_ALGO_TWOSHOT ? 1 : 0; // two-shot: each non-root moves one slice
  const int blocks = grid_for(mode ? nvec / (size_t)(n - 1) + 1 : nvec, 4);
  return with_unit(off | bytes, [&](auto u) { return launch_coll(bcast_kernel<decltype(u), 4>, "bcast_kernel", sig, blocks, kThreads, 0, s, off, bytes, root, mode); });
}

static int launch_allgather(int algo, int dtype, size_t count, uint64_t in_off, uint64_t out_off, size_t bytes, cudaStream_t s, size_t total = 0) {
  const uint64_t sig = make_sig(2, dtype, 0, algo, count, total);
  const int blocks = grid_for(bytes / 16 + 1, 4);
  if (algo == B200MPI_ALGO_NVLS) return launch_coll(allgather_nvls_kernel<4>, "allgather_nvls_kernel", sig, blocks, kThreads, 0, s, in_off, out_off, bytes);
  return with_unit(in_off | out_off | bytes, [&](auto u) {
    using U = decltype(u);
    if (algo == B200MPI_ALGO_RING) return launch_coll(allgather_ring_kernel<U>, "allgather kernel", sig, blocks, kThreads, 0, s, in_off, out_off, bytes);
    return launch_coll(allgather_push_kernel<U, 4>, "allgather kernel", sig, blocks, kThreads, 0, s, in_off, out_off, bytes);
  });
}

// ---------------------------------------------------------------------------------------------
// buffer resolution: heap-resident device memory is used in place; anything else (host slices,
// foreign device pointers) is staged through a heap block on the collective stream, block 0 for
// the send side and block 1 for the recv side.
// ---------------------------------------------------------------------------------------------
static int ensure_stage(int which, size_t bytes) {
  if (g->stage_len[which] >= bytes && bytes > 0) return 0;
  if (g->stage_len[which]) {
    // the previous block may still be in use by enqueued work
    cudaStreamSynchronize(g->stream);
    g->heap.free_off(g->stage_off[which]);
    g->stage_len[which] = 0;
  }
  size_t off = 0;
  size_t want = std::max<size_t>(bytes, 1u << 20);
  if (g->heap.alloc(want, off)) return fail(B200MPI_ERR_NOMEM, "symmetric heap exhausted while staging " + std::to_string(bytes) + " bytes (raise B200MPI_HEAP_BYTES)");
  g->stage_off[which] = off;
  g->stage_len[which] = want;
  return 0;
}

struct Buf {
  uint64_t off = 0;
  bool staged = false;
};

// True when [p, p + bytes) is memory of this rank's GPU: its own heap, or a buffer the runtime
// reports as device memory on g->dev (not a peer's memory, not managed or host memory).
static bool on_this_gpu(const void* p, size_t bytes) {
  size_t off;
  if (g->heap.contains(p, bytes, off)) return true;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { (void)cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeDevice && a.device == g->dev;
}

// Device-to-device copy between a caller's buffer `foreign` and a staging area in this rank's heap.
static int stage_copy(void* dst, const void* src, size_t bytes, const void* foreign) {
  return on_this_gpu(foreign, bytes) ? launch_local_copy(dst, src, bytes, g->stream) : launch_copy(dst, src, bytes, g->stream);
}

// [p, p + bytes) as an offset in this rank's heap: where it lies, or staging block `which`, which is
// filled from p when `fill`.
static int resolve(const void* p, size_t bytes, int memkind, int which, bool fill, Buf& b) {
  size_t off;
  if (memkind == B200MPI_DEVICE && g->heap.contains(p, bytes, off)) {
    b = {off, false};
    return 0;
  }
  const int rc = ensure_stage(which, bytes);
  if (rc) return rc;
  b = {g->stage_off[which], true};
  if (!fill || bytes == 0) return 0;
  char* dst = (char*)g->heap.base[g->ctrl.rank] + b.off;
  if (memkind == B200MPI_HOST) CUDA_OK(cudaMemcpyAsync(dst, p, bytes, cudaMemcpyHostToDevice, g->stream));
  else return stage_copy(dst, p, bytes, p);
  return 0;
}

// How a collective's two buffers lie on this rank.
enum Layout {
  kApart,      // separate buffers
  kSendOnly,   // this rank's recv is not written (Bcast root, Reduce and Gatherv off root)
  kRecvOnly,   // this rank's send is not read (Bcast and Scatterv off root)
  kRecvInSend, // in place: recv lies `at` bytes into send
  kSendInRecv, // in place: send lies `at` bytes into recv
};

// The heap offsets a collective's kernel reads this rank's send from (`in`) and writes its recv to
// (`out`), and the caller's recv that finish copies `out` back to when it is staged.
struct Staging {
  uint64_t in = 0, out = 0;
  void* recv = nullptr; // nullptr: nothing to copy back
  size_t rbytes = 0;
  int memkind = 0;
};

// Resolves a call's send side (read by this rank) and recv side (written by this rank) to heap
// offsets.  A side this rank does not use announces the other side's offset; no peer reads or writes
// it there.  In place, the inner buffer shares the outer one's staging only when the outer one is
// the send side, because only the send side's staging is filled from the caller: a send inside a
// staged recv is staged on its own.
static int stage(Staging& st, int memkind, const void* send, size_t sbytes, void* recv, size_t rbytes, Layout lay = kApart, size_t at = 0) {
  Buf in, out;
  int rc;
  if (lay == kSendInRecv) {
    if ((rc = resolve(recv, rbytes, memkind, 1, false, out))) return rc;
    if (!out.staged) in.off = out.off + at;
    else if ((rc = resolve(send, sbytes, memkind, 0, true, in))) return rc;
  } else {
    if (lay != kRecvOnly && (rc = resolve(send, sbytes, memkind, 0, true, in))) return rc;
    if (lay == kRecvInSend) out = {in.off + at, in.staged};
    else if (lay == kSendOnly) out.off = in.off;
    else if ((rc = resolve(recv, rbytes, memkind, 1, false, out))) return rc;
    if (lay == kRecvOnly) in.off = out.off;
  }
  st = {in.off, out.off, out.staged ? recv : nullptr, rbytes, memkind};
  return 0;
}

// Ends a call on the collective stream.  A staged recv is copied back after the kernel; a
// synchronous call first waits and copies only when the status word says the call succeeded, so a
// mismatched call (B200MPI_ERR_PEER) leaves the caller's buffer untouched, as on the heap.  The
// _async entries enqueue the copy-back without waiting: they take only DEVICE memory, and
// b200mpi_stream_sync reports their status (a staged recv of a failed _async call is overwritten).
static int finish(bool async, const Staging& st = {}) {
  if (st.recv && st.rbytes) {
    if (!async) {
      CUDA_OK(cudaStreamSynchronize(g->stream));
      const int rc = check_status();
      if (rc) return rc;
    }
    const char* src = (const char*)g->heap.base[g->ctrl.rank] + st.out;
    if (st.memkind == B200MPI_HOST) CUDA_OK(cudaMemcpyAsync(st.recv, src, st.rbytes, cudaMemcpyDeviceToHost, g->stream));
    else if (const int rc = stage_copy(st.recv, src, st.rbytes, st.recv)) return rc;
  }
  if (async) return 0;
  CUDA_OK(cudaStreamSynchronize(g->stream));
  return check_status();
}

static int local_copy(void* dst, const void* src, size_t bytes, int memkind, bool async) {
  if (dst == src || bytes == 0) return finish(async);
  if (memkind == B200MPI_HOST) {
    // world of one: the value still makes the round trip through the device (no CPU data path)
    const int rc = ensure_stage(0, bytes);
    if (rc) return rc;
    char* st = (char*)g->heap.base[g->ctrl.rank] + g->stage_off[0];
    CUDA_OK(cudaMemcpyAsync(st, src, bytes, cudaMemcpyHostToDevice, g->stream));
    CUDA_OK(cudaMemcpyAsync(dst, st, bytes, cudaMemcpyDeviceToHost, g->stream));
  } else {
    const bool local = on_this_gpu(dst, bytes) && on_this_gpu(src, bytes);
    int rc = local ? launch_local_copy(dst, src, bytes, g->stream) : launch_copy(dst, src, bytes, g->stream);
    if (rc) return rc;
  }
  return finish(async);
}

// A device-wide rendezvous with nothing in between, on `s`.
static int launch_barrier(cudaStream_t s) { return launch_coll(barrier_kernel, "barrier_kernel", make_sig(3, 0, 0, 0, 0), 1, 32, 0, s); }

// The LL sequence has crossed 2^32 (ll_seq_next): a lane cell may already hold the value about to be
// issued, zeros from Init or a value written 2^32 calls ago.  A barrier (no peer is still pushing cells
// of an earlier call), this rank's lanes of both parities cleared, a second barrier (no peer pushes
// its next cells before they are clear).  ll_seq agrees on every rank, so every rank comes here on
// the same call, once per 2^32 LL calls.
static int clear_ll_lanes(cudaStream_t s) {
  int rc = launch_barrier(s);
  if (rc) return rc;
  CUDA_OK(cudaMemsetAsync((char*)g->heap.base[g->ctrl.rank] + kLLOff, 0, kLLRegionCells * sizeof(uint4), s));
  rc = launch_barrier(s);
  if (rc) return rc;
  g->ll_wrap_pending = false;
  return 0;
}

// Barrier-free LL allreduce for small messages (kernels.cuh): any local device pointers.
template <typename T, typename Op>
static int launch_ll_t(const void* send, void* recv, size_t count, uint32_t* done_host, cudaStream_t s) {
  Comm c = g->comm;
  const LLSeqNext next = ll_seq_next(g->ll_seq, 1);
  if (next.wrapped || g->ll_wrap_pending) {
    const int rc = clear_ll_lanes(s);
    if (rc) return rc;
  }
  const uint32_t seq = g->ll_seq = next.seq;
  const size_t ncell = (count * sizeof(T) + 7) / 8;
  const int blocks = (int)std::max<size_t>(1, std::min<size_t>((ncell + 255) / 256, 128)); // one cell per thread up to 256 KiB
  allreduce_ll_kernel<T, Op><<<blocks, 256, 0, s>>>(c, (const T*)send, (T*)recv, count, seq, done_host);
  return launch_check("allreduce_ll_kernel");
}
static int launch_ll(int dtype, int op, const void* send, void* recv, size_t count, uint32_t* done_host, cudaStream_t s) {
  return with_reduction(
      dtype, op, [&](auto t, auto o) { return launch_ll_t<decltype(t), decltype(o)>(send, recv, count, done_host, s); },
      [] { return fail(B200MPI_ERR_UNSUPPORTED, "allreduce(LL): unsupported dtype/op"); });
}

// Small host-slice Allreduce: memcpy into a device-mapped pinned buffer, ONE kernel that loads its
// input over PCIe and stores result and completion word into host memory, spin on that word (no
// H2D / D2H copies, no stream synchronisation), memcpy out.
static int allreduce_ll_host(const void* send, void* recv, size_t count, int dtype, int op) {
  const size_t bytes = count * esize(dtype);
  const size_t half = kLLRegionCells / 4 * 8; // the largest message of any world size (n = 2)
  if (!g->ll_host) {
    CUDA_OK(cudaHostAlloc((void**)&g->ll_host, 2 * half + 64, cudaHostAllocMapped));
    CUDA_OK(cudaHostGetDevicePointer((void**)&g->ll_dev, g->ll_host, 0));
    *(volatile uint32_t*)(g->ll_host + 2 * half) = 0;
  }
  CUDA_OK(cudaStreamSynchronize(g->stream)); // enqueue-only calls issued earlier may still be running
  if (bytes) memcpy(g->ll_host, send, bytes);
  volatile uint32_t* done = (volatile uint32_t*)(g->ll_host + 2 * half);
  *done = 0; // no sequence number is 0: the word cannot match before this call's kernel writes it
             // (after a restart of the sequence it may still hold this call's value from 2^32 calls ago)
  int rc = launch_ll(dtype, op, g->ll_dev, g->ll_dev + half, count, (uint32_t*)(g->ll_dev + 2 * half), g->stream);
  if (rc) return rc;
  const uint32_t seq = g->ll_seq;
  Spinner sp(g->watchdog_ns + 5000000000ll);
  while (*done != seq) {
    if (*(volatile uint32_t*)g->status_host) break; // device-side watchdog fired
    if (!sp.step()) break;
  }
  if (*done != seq) {
    cudaStreamSynchronize(g->stream);
    rc = check_status();
    return rc ? rc : fail(B200MPI_ERR_TIMEOUT, "allreduce(LL): kernel did not complete");
  }
  std::atomic_thread_fence(std::memory_order_acquire);
  if (bytes) memcpy(recv, g->ll_host + half, bytes);
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Host slices (what an unmodified Go caller passes, bounce.go:120-127): H2D, collective and D2H
// are pipelined in chunks over three streams so PCIe runs in both directions while the GPUs talk.
// Every rank derives the same chunking from (count, dtype, n) and the knobs, whatever memory its own
// buffer lives in (pipe_chunk_elems), so the per-chunk collectives line up; the signature of each
// chunk also carries the total count.
//   pinned (cudaHostAlloc / cudaHostRegister'ed) memory: DMA straight from / to the caller's buffer;
//   pageable memory (a Go slice, a numpy array): through a ring of pinned bounce chunks filled and
//   drained by the helper threads of CopyPool while the DMA engines work on the neighbours.
// ---------------------------------------------------------------------------------------------
// True when [p, p + bytes) may be DMA'd in place.  A range this rank registered counts only when one
// registration holds all of it: a neighbour of a registered buffer can start in the page they share,
// and a copy that starts there runs past the registration (cudaErrorInvalidValue).
static bool is_pinned(const void* p, size_t bytes) {
  if (!p || bytes == 0) return true;
  const uintptr_t a0 = (uintptr_t)p, a1 = a0 + bytes;
  for (const auto& e : g->registered)
    if (a0 < e.first + e.second && e.first < a1) return a0 >= e.first && a1 <= e.first + e.second;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { (void)cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}

static bool ensure_registered(const void* p, size_t bytes) {
  if (!p || bytes == 0) return true;
  const uintptr_t page = 4096;
  uintptr_t lo = (uintptr_t)p & ~(page - 1), hi = ((uintptr_t)p + bytes + page - 1) & ~(page - 1);
  for (size_t i = 0; i < g->registered.size(); ++i) {
    auto e = g->registered[i];
    if (lo >= e.first && hi <= e.first + e.second) {
      g->registered.erase(g->registered.begin() + i);
      g->registered.push_back(e);
      return true;
    }
  }
  // replace entries the new range overlaps (the caller re-used part of an old buffer, or a neighbour
  // shares a page with it) by one registration of the union, so that the buffers they held stay
  // covered; drop the oldest beyond 16
  for (size_t i = 0; i < g->registered.size();) {
    auto e = g->registered[i];
    if (lo < e.first + e.second && e.first < hi) {
      cudaHostUnregister((void*)e.first);
      g->registered.erase(g->registered.begin() + i);
      lo = std::min(lo, e.first);
      hi = std::max(hi, e.first + e.second);
      i = 0; // the union may reach entries already passed
    } else {
      ++i;
    }
  }
  while (g->registered.size() >= 16) { cudaHostUnregister((void*)g->registered.front().first); g->registered.erase(g->registered.begin()); }
  if (cudaHostRegister((void*)lo, hi - lo, cudaHostRegisterDefault) != cudaSuccess) { (void)cudaGetLastError(); return false; }
  g->registered.push_back({lo, hi - lo});
  return true;
}

struct PipeSpec {
  int coll;          // B200MPI_COLL_ALLREDUCE / _BCAST / _ALLGATHER
  int dtype, op, root;
  size_t count;      // elements (per rank for allgather)
  const char* in;    // host input of this rank (nullptr: none, e.g. a bcast non-root)
  char* out;         // host output of this rank (nullptr: none, e.g. the bcast root)
};

static int ensure_bounce(size_t chunk) {
  if (g->bounce && g->bounce_chunk >= chunk) return 0;
  if (g->bounce) { cudaFreeHost(g->bounce); g->bounce = nullptr; }
  void* p = nullptr;
  int rc = numa_host_alloc(2 * (size_t)Ctx::kBounceSlots * chunk, &p);
  if (rc) return rc;
  g->bounce = (char*)p;
  g->bounce_chunk = chunk;
  if (!g->pool.running()) g->pool.start(g->host_threads, g->gpu_numa_node);
  return 0;
}

static int host_pipeline(const PipeSpec& sp) {
  const size_t es = esize(sp.dtype), B = sp.count * es;
  const int n = g->ctrl.n, R = Ctx::kBounceSlots;
  const bool ag = sp.coll == B200MPI_COLL_ALLGATHER;
  const size_t rows = ag ? (size_t)n : 1;
  const size_t in_bytes = sp.in ? B : 0, out_bytes = sp.out ? B * rows : 0;
  bool pinned = is_pinned(sp.in, in_bytes) && is_pinned(sp.out, out_bytes);
  if (!pinned && g->host_register)
    pinned = (is_pinned(sp.in, in_bytes) || ensure_registered(sp.in, in_bytes)) && (is_pinned(sp.out, out_bytes) || ensure_registered(sp.out, out_bytes));
  const bool bounce = !pinned && g->host_threads > 0;
  const size_t chunk_elems = pipe_chunk_elems(es, rows, n, bounce, g->pipe_chunk_bytes, g->bounce_chunk_bytes);
  const size_t nch = (sp.count + chunk_elems - 1) / chunk_elems;
  int rc = ensure_stage(0, B);
  if (rc) return rc;
  if (ag && n > 1 && (rc = ensure_stage(1, B * n))) return rc;
  if (bounce && (rc = ensure_bounce(chunk_elems * es * rows))) return rc;
  char* heap = (char*)g->heap.base[g->ctrl.rank];
  char* st_in = heap + g->stage_off[0];
  char* st_out = (ag && n > 1) ? heap + g->stage_off[1] : st_in; // world of one: recv block 0 is the send block
  while (g->pipe_events.size() < 3 * nch) {
    cudaEvent_t e;
    CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    g->pipe_events.push_back(e);
  }
  CUDA_OK(cudaStreamSynchronize(g->stream)); // earlier work may still use the staging blocks
  char* b_in = g->bounce;
  char* b_out = g->bounce ? g->bounce + (size_t)R * g->bounce_chunk : nullptr;
  std::atomic<int> pend_in[Ctx::kBounceSlots], pend_out[Ctx::kBounceSlots];
  for (int i = 0; i < R; ++i) { pend_in[i].store(0); pend_out[i].store(0); }
  // queued copy tasks point at these counters: whatever way this function is left (CUDA error paths
  // included), the helper threads are done with them first
  struct Drain {
    CopyPool& pool; std::atomic<int>* a; std::atomic<int>* b; int n; bool on;
    ~Drain() { if (on) for (int i = 0; i < n; ++i) { pool.wait(a[i]); pool.wait(b[i]); } }
  } drain{g->pool, pend_in, pend_out, R, bounce};
  auto lo_of = [&](size_t k) { return k * chunk_elems; };
  auto len_of = [&](size_t k) { return std::min(chunk_elems, sp.count - lo_of(k)); };

  // GPU side of chunk k: H2D, collective, D2H (enqueue only)
  auto gpu_stage = [&](size_t k) -> int {
    const size_t lo = lo_of(k) * es, len = len_of(k) * es;
    cudaEvent_t e_in = g->pipe_events[3 * k], e_coll = g->pipe_events[3 * k + 1], e_out = g->pipe_events[3 * k + 2];
    bool have_in = false;
    if (sp.in) {
      const char* src = sp.in + lo;
      if (bounce) { g->pool.wait(pend_in[k % R]); src = b_in + (k % R) * g->bounce_chunk; }
      CUDA_OK(cudaMemcpyAsync(st_in + lo, src, len, cudaMemcpyHostToDevice, g->h2d_stream));
      CUDA_OK(cudaEventRecord(e_in, g->h2d_stream));
      have_in = true;
    }
    cudaEvent_t ready = e_in;
    if (n > 1) {
      if (have_in) CUDA_OK(cudaStreamWaitEvent(g->stream, e_in, 0));
      const uint64_t off = g->stage_off[0] + lo;
      int r2;
      if (sp.coll == B200MPI_COLL_ALLREDUCE) r2 = launch_allreduce(pick_allreduce(len, sp.dtype, sp.op, true), sp.dtype, sp.op, off, off, len_of(k), g->stream, sp.count);
      else if (sp.coll == B200MPI_COLL_BCAST) r2 = launch_bcast(pick_bcast(len), sp.dtype, len_of(k), off, len, sp.root, g->stream, sp.count);
      else r2 = launch_allgather(pick_allgather(len), sp.dtype, len_of(k), off, g->stage_off[1] + lo * n, len, g->stream, sp.count);
      if (r2) return r2;
      CUDA_OK(cudaEventRecord(e_coll, g->stream));
      ready = e_coll;
    }
    if (sp.out) {
      if (n > 1 || have_in) CUDA_OK(cudaStreamWaitEvent(g->d2h_stream, ready, 0));
      const char* src = st_out + (ag && n > 1 ? lo * n : lo);
      if (bounce) {
        g->pool.wait(pend_out[k % R]); // the copy-out that used this slot R chunks ago
        CUDA_OK(cudaMemcpyAsync(b_out + (k % R) * g->bounce_chunk, src, len * rows, cudaMemcpyDeviceToHost, g->d2h_stream));
      } else if (rows == 1) {
        CUDA_OK(cudaMemcpyAsync(sp.out + lo, src, len, cudaMemcpyDeviceToHost, g->d2h_stream));
      } else { // allgather: n rows of len bytes, B apart in the caller's recv buffer
        CUDA_OK(cudaMemcpy2DAsync(sp.out + lo, B, src, len, len, rows, cudaMemcpyDeviceToHost, g->d2h_stream));
      }
      CUDA_OK(cudaEventRecord(e_out, g->d2h_stream));
    }
    return 0;
  };
  // host side after the D2H of chunk k (bounce only): scatter the chunk into the caller's buffer
  auto host_out = [&](size_t k) -> int {
    if (!bounce || !sp.out) return 0;
    CUDA_OK(cudaEventSynchronize(g->pipe_events[3 * k + 2]));
    const size_t lo = lo_of(k) * es, len = len_of(k) * es;
    for (size_t r = 0; r < rows; ++r) g->pool.submit(sp.out + r * B + lo, b_out + (k % R) * g->bounce_chunk + r * len, len, pend_out[k % R]);
    return 0;
  };
  const size_t lag = 2; // chunks between issuing the D2H of a chunk and draining its bounce slot
  size_t next_gpu = 0, next_out = 0; // next chunk whose GPU stage / host-side drain is due
  for (size_t k = 0; k < nch; ++k) {
    if (bounce && sp.in) {
      // the H2D that read this bounce slot R chunks ago (issued: next_gpu >= k-1 > k-R)
      if (k >= (size_t)R) CUDA_OK(cudaEventSynchronize(g->pipe_events[3 * (k - R)]));
      g->pool.submit(b_in + (k % R) * g->bounce_chunk, sp.in + lo_of(k) * es, len_of(k) * es, pend_in[k % R]);
      while (next_gpu < k) // the helper threads fill chunk k while the GPU works on chunk k-1
        if ((rc = gpu_stage(next_gpu++))) return rc;
    } else {
      if ((rc = gpu_stage(k))) return rc;
      next_gpu = k + 1;
    }
    while (next_out + lag < next_gpu)
      if ((rc = host_out(next_out++))) return rc;
  }
  while (next_gpu < nch)
    if ((rc = gpu_stage(next_gpu++))) return rc;
  while (next_out < nch)
    if ((rc = host_out(next_out++))) return rc;
  if (bounce && sp.out)
    for (int i = 0; i < R; ++i) g->pool.wait(pend_out[i]);
  CUDA_OK(cudaStreamSynchronize(g->d2h_stream));
  CUDA_OK(cudaStreamSynchronize(g->h2d_stream));
  CUDA_OK(cudaStreamSynchronize(g->stream));
  return check_status();
}

// What every collective checks first, in this order: the data plane, the dtype (a reduction refuses
// u8 and unknown types as unsupported), a reduction's op, a rooted call's root and the memory kind.
// es receives the element size.  Each call then checks its own NULL-buffer and in-place rules.
enum { kReduces = 1, kRooted = 2 };
static int check_coll(const char* what, int traits, int dtype, int op, int root, int memkind, size_t& es) {
  int rc = need_data_plane();
  if (rc) return rc;
  auto arg = [&](const char* msg) { return fail(B200MPI_ERR_ARG, std::string(what) + ": " + msg); };
  es = esize(dtype);
  if ((traits & kReduces) && (es == 0 || dtype == B200MPI_U8)) return fail(B200MPI_ERR_UNSUPPORTED, std::string(what) + ": dtype must be f32, f64 or i64");
  if (es == 0) return arg("unknown dtype");
  if ((traits & kReduces) && (op < B200MPI_SUM || op > B200MPI_MIN)) return arg("unknown op");
  if ((traits & kRooted) && (root < 0 || root >= g->ctrl.n)) return arg("root out of range");
  if (memkind != B200MPI_HOST && memkind != B200MPI_DEVICE) return arg("bad memkind");
  return 0;
}
static int null_buffer(const char* what) { return fail(B200MPI_ERR_ARG, std::string(what) + ": NULL buffer with count > 0"); }

static int do_allreduce(const void* send, void* recv, size_t count, int dtype, int op, int memkind, bool async) {
  size_t es;
  int rc = check_coll("allreduce", kReduces, dtype, op, 0, memkind, es);
  if (rc) return rc;
  if (count && (!send || !recv)) return null_buffer("allreduce");
  const size_t bytes = count * es;
  if (memkind == B200MPI_HOST && !async && bytes >= g->pipe_min_bytes) {
    PipeSpec sp = {B200MPI_COLL_ALLREDUCE, dtype, op, 0, count, (const char*)send, (char*)recv};
    return host_pipeline(sp);
  }
  if (g->ctrl.n == 1) return local_copy(recv, send, bytes, memkind, async);
  const int algo = pick_allreduce(bytes, dtype, op);
  if (algo == B200MPI_ALGO_LL) {
    // any local device pointer works (peers never read it)
    if (memkind == B200MPI_DEVICE) {
      rc = launch_ll(dtype, op, send, recv, count, nullptr, g->stream);
      return rc ? rc : finish(async);
    }
    return allreduce_ll_host(send, recv, count, dtype, op);
  }
  Staging st;
  if ((rc = stage(st, memkind, send, bytes, recv, bytes, send == recv ? kRecvInSend : kApart))) return rc;
  if ((rc = launch_allreduce(algo, dtype, op, st.in, st.out, count, g->stream))) return rc;
  return finish(async, st);
}

static int do_bcast(void* buf, size_t count, int dtype, int root, int memkind, bool async) {
  size_t es;
  int rc = check_coll("bcast", kRooted, dtype, 0, root, memkind, es);
  if (rc) return rc;
  if (count && !buf) return null_buffer("bcast");
  if (g->ctrl.n == 1) return finish(async);
  const size_t bytes = count * es;
  const bool is_root = g->ctrl.rank == root;
  if (memkind == B200MPI_HOST && !async && bytes >= g->pipe_min_bytes) {
    PipeSpec sp = {B200MPI_COLL_BCAST, dtype, 0, root, count, is_root ? (const char*)buf : nullptr, is_root ? nullptr : (char*)buf};
    return host_pipeline(sp);
  }
  Staging st;
  if ((rc = stage(st, memkind, buf, bytes, buf, bytes, is_root ? kSendOnly : kRecvOnly))) return rc;
  if ((rc = launch_bcast(pick_bcast(bytes), dtype, count, st.in, bytes, root, g->stream))) return rc;
  return finish(async, st);
}

static int do_allgather(const void* send, void* recv, size_t count, int dtype, int memkind, bool async) {
  size_t es;
  int rc = check_coll("allgather", 0, dtype, 0, 0, memkind, es);
  if (rc) return rc;
  if (count && (!send || !recv)) return null_buffer("allgather");
  const size_t bytes = count * es;
  const int n = g->ctrl.n;
  if (memkind == B200MPI_HOST && !async && bytes * n >= g->pipe_min_bytes) {
    PipeSpec sp = {B200MPI_COLL_ALLGATHER, dtype, 0, 0, count, (const char*)send, (char*)recv};
    return host_pipeline(sp);
  }
  if (n == 1) return local_copy(recv, send, bytes, memkind, async);
  const size_t at = (size_t)g->ctrl.rank * bytes;
  Staging st;
  if ((rc = stage(st, memkind, send, bytes, recv, bytes * n, (const char*)send == (const char*)recv + at ? kSendInRecv : kApart, at))) return rc;
  if ((rc = launch_allgather(pick_allgather(bytes), dtype, count, st.in, st.out, bytes, g->stream))) return rc;
  return finish(async, st);
}

// ReduceScatter: send holds size()*count elements (block j is reduced onto rank j), recv holds count.
static int do_reduce_scatter(const void* send, void* recv, size_t count, int dtype, int op, int memkind, bool async) {
  size_t es;
  int rc = check_coll("reduce_scatter", kReduces, dtype, op, 0, memkind, es);
  if (rc) return rc;
  if (count && (!send || !recv)) return null_buffer("reduce_scatter");
  const size_t bytes = count * es;
  const int n = g->ctrl.n;
  if (n == 1) return local_copy(recv, send, bytes, memkind, async);
  const size_t at = (size_t)g->ctrl.rank * bytes;
  Staging st;
  if ((rc = stage(st, memkind, send, bytes * n, recv, bytes, (const char*)recv == (const char*)send + at ? kRecvInSend : kApart, at))) return rc;
  if ((rc = launch_reduce_scatter(pick_reduce_scatter(bytes, dtype, op), dtype, op, st.in, st.out, count, g->stream))) return rc;
  return finish(async, st);
}

// Reduce: like Allreduce but only `root`'s recv is written (recv may be NULL elsewhere).
static int do_reduce(const void* send, void* recv, size_t count, int dtype, int op, int root, int memkind, bool async) {
  size_t es;
  int rc = check_coll("reduce", kReduces | kRooted, dtype, op, root, memkind, es);
  if (rc) return rc;
  const int n = g->ctrl.n;
  const bool is_root = g->ctrl.rank == root;
  if (count && (!send || (is_root && !recv))) return null_buffer("reduce");
  const size_t bytes = count * es;
  if (n == 1) return local_copy(recv, send, bytes, memkind, async);
  Staging st;
  if ((rc = stage(st, memkind, send, bytes, recv, bytes, !is_root ? kSendOnly : recv == send ? kRecvInSend : kApart))) return rc;
  int algo = g->algo[B200MPI_COLL_ALLREDUCE] == B200MPI_ALGO_TWOSHOT ? B200MPI_ALGO_TWOSHOT
             : (g->heap.mc_base && nvls_supports(dtype, op) && n >= g->nvls_min_ranks) ? B200MPI_ALGO_NVLS : B200MPI_ALGO_TWOSHOT;
  if ((rc = launch_reduce(algo, dtype, op, st.in, st.out, count, root, g->stream))) return rc;
  return finish(async, st);
}

// Scan: rank r's recv = send_0 op ... op send_r, in rank order.  Exscan (exclusive): the same up to
// send_{r-1}; rank 0's recv is not written and may be NULL.  One algorithm, no host pipelining: host
// slices and foreign device pointers are staged whole.
static int do_scan(const void* send, void* recv, size_t count, int dtype, int op, int memkind, bool exclusive) {
  const char* what = exclusive ? "exscan" : "scan";
  size_t es;
  int rc = check_coll(what, kReduces, dtype, op, 0, memkind, es);
  if (rc) return rc;
  const bool gets = !exclusive || g->ctrl.rank > 0; // this rank's recv is written
  if (count && (!send || (gets && !recv))) return null_buffer(what);
  const size_t bytes = count * es;
  if (g->ctrl.n == 1) return gets ? local_copy(recv, send, bytes, memkind, false) : finish(false);
  Staging st;
  if ((rc = stage(st, memkind, send, bytes, recv, bytes, !gets ? kSendOnly : recv == send ? kRecvInSend : kApart))) return rc;
  if ((rc = launch_scan(exclusive, dtype, op, st.in, st.out, count, g->stream))) return rc;
  return finish(false, st);
}

// MAXLOC / MINLOC over `count` 16-byte {value, int64 loc} pairs whose value type is `dtype`: into
// every rank's recv (all) or into root's only, where recv may be NULL elsewhere.  One algorithm, no
// host pipelining: host slices and foreign device pointers are staged whole.
static int do_allreduce_loc(const void* send, void* recv, size_t count, int dtype, int op, int root, int memkind, bool all) {
  const char* what = all ? "allreduce_loc" : "reduce_loc";
  size_t es;
  int rc = check_coll(what, all ? kReduces : kReduces | kRooted, dtype, op, root, memkind, es);
  if (rc) return rc;
  if (op == B200MPI_SUM) return fail(B200MPI_ERR_UNSUPPORTED, std::string(what) + ": op must be max (MAXLOC) or min (MINLOC)");
  const bool gets = all || g->ctrl.rank == root; // this rank's recv is written
  if (count && (!send || (gets && !recv))) return null_buffer(what);
  if (((uintptr_t)send | (gets ? (uintptr_t)recv : 0)) & 7) return fail(B200MPI_ERR_ARG, std::string(what) + ": pair buffers must be 8-byte aligned");
  const size_t bytes = count * sizeof(Loc<double>);
  if (g->ctrl.n == 1) return local_copy(recv, send, bytes, memkind, false);
  Staging st;
  if ((rc = stage(st, memkind, send, bytes, recv, bytes, !gets ? kSendOnly : recv == send ? kRecvInSend : kApart))) return rc;
  if ((rc = launch_allreduce_loc(dtype, op, st.in, st.out, count, all ? -1 : root, g->stream))) return rc;
  return finish(false, st);
}

// Alltoall: send and recv hold size()*count elements; block j of send goes to rank j's block rank().
static int do_alltoall(const void* send, void* recv, size_t count, int dtype, int memkind, bool async) {
  size_t es;
  int rc = check_coll("alltoall", 0, dtype, 0, 0, memkind, es);
  if (rc) return rc;
  if (count && (!send || !recv)) return null_buffer("alltoall");
  if (send == recv && count) return fail(B200MPI_ERR_ARG, "alltoall: in place is not supported");
  const size_t bytes = count * es;
  const int n = g->ctrl.n;
  if (n == 1) return local_copy(recv, send, bytes, memkind, async);
  Staging st;
  if ((rc = stage(st, memkind, send, bytes * n, recv, bytes * n))) return rc;
  const uint64_t sig = make_sig(6, dtype, 0, 0, count);
  const int blocks = grid_for(bytes / 16 + 1, 4);
  rc = with_unit(st.in | st.out | bytes, [&](auto u) { return launch_coll(alltoall_kernel<decltype(u), 4>, "alltoall_kernel", sig, blocks, kThreads, 0, g->stream, st.in, st.out, bytes); });
  return rc ? rc : finish(async, st);
}

// ---------------------------------------------------------------------------------------------
// Gather(v), Scatter(v), Allgatherv: blocks of counts[r] elements packed in rank order.  One
// algorithm each, no host pipelining: host slices and foreign device pointers are staged whole.
// ---------------------------------------------------------------------------------------------
// counts[n] -> byte displacements, and a hash of the whole table for the call signature (order
// matters: tables that differ by a swap of two counts hash differently).
static int make_vtable(const char* what, const size_t* counts, size_t es, VTable& vt, uint64_t& hash) {
  const int n = g->ctrl.n;
  if (!counts) return fail(B200MPI_ERR_ARG, std::string(what) + ": NULL counts table");
  uint64_t off = 0;
  hash = 0x76746162ull;
  for (int r = 0; r < n; ++r) {
    vt.off[r] = off;
    if (counts[r] > (SIZE_MAX - off) / es) return fail(B200MPI_ERR_ARG, std::string(what) + ": sum(counts) * element size overflows");
    off += counts[r] * es;
    hash = mix64(hash ^ (counts[r] + 0x9e3779b97f4a7c15ull * (uint64_t)(r + 1)));
  }
  for (int r = n; r <= kMaxRanks; ++r) vt.off[r] = off;
  return 0;
}

// The grid of a table-driven launch follows the largest block, so every rank launches the same one.
static int vtable_grid(const VTable& vt, int unroll = 4) {
  size_t largest = 0;
  for (int r = 0; r < g->ctrl.n; ++r) largest = std::max<size_t>(largest, vt.off[r + 1] - vt.off[r]);
  return grid_for(largest / 16 + 1, unroll);
}

// OR of the displacements off[0..n]: with this rank's offsets they pick its access unit (with_unit).
static uint64_t vtable_bits(const VTable& vt) {
  uint64_t m = 0;
  for (int r = 0; r <= g->ctrl.n; ++r) m |= vt.off[r];
  return m;
}

// Gatherv: rank r's send lands at displacement r of root's recv; recv may be NULL off root.
// Allgatherv (all): it lands at displacement r of every rank's recv.
static int do_gatherv(const void* send, void* recv, const size_t* counts, int dtype, int root, bool all, int memkind) {
  const char* what = all ? "allgatherv" : "gatherv";
  size_t es;
  int rc = check_coll(what, all ? 0 : kRooted, dtype, 0, root, memkind, es);
  if (rc) return rc;
  if (all) root = -1;
  const int n = g->ctrl.n, me = g->ctrl.rank;
  VTable vt;
  uint64_t hash;
  if ((rc = make_vtable(what, counts, es, vt, hash))) return rc;
  const size_t mine = vt.off[me + 1] - vt.off[me], total = vt.off[n];
  const bool gets = all || me == root; // this rank's recv is written
  if ((mine && !send) || (gets && total && !recv)) return null_buffer(what);
  if (n == 1) return local_copy(recv, send, total, memkind, false);
  const bool inplace = gets && recv && (const char*)send == (const char*)recv + vt.off[me];
  Staging st; // off root the recv is announced but never written: only root's recv is a destination
  if ((rc = stage(st, memkind, send, mine, recv, total, !gets ? kSendOnly : inplace ? kSendInRecv : kApart, vt.off[me]))) return rc;
  const uint64_t sig = make_sig(all ? 9 : 7, dtype, root, 0, total / es, hash);
  const int blocks = vtable_grid(vt);
  rc = with_unit(st.in | st.out | vtable_bits(vt), [&](auto u) {
    return launch_coll(gatherv_push_kernel<decltype(u), 4>, "gatherv_push_kernel", sig, blocks, kThreads, 0, g->stream, st.in, st.out, vt, root);
  });
  return rc ? rc : finish(false, st);
}

// Scatterv: block r of root's send (NULL allowed off root) goes to rank r's recv.
static int do_scatterv(const void* send, void* recv, const size_t* counts, int dtype, int root, int memkind) {
  size_t es;
  int rc = check_coll("scatterv", kRooted, dtype, 0, root, memkind, es);
  if (rc) return rc;
  const int n = g->ctrl.n, me = g->ctrl.rank;
  VTable vt;
  uint64_t hash;
  if ((rc = make_vtable("scatterv", counts, es, vt, hash))) return rc;
  const size_t mine = vt.off[me + 1] - vt.off[me], total = vt.off[n];
  const bool is_root = me == root;
  if ((mine && !recv) || (is_root && total && !send)) return null_buffer("scatterv");
  if (n == 1) return local_copy(recv, send, total, memkind, false);
  const bool inplace = is_root && send && (const char*)recv == (const char*)send + vt.off[me];
  Staging st; // off root the send is announced but never read: only root's send is a source
  if ((rc = stage(st, memkind, send, total, recv, mine, !is_root ? kRecvOnly : inplace ? kRecvInSend : kApart, vt.off[me]))) return rc;
  const uint64_t sig = make_sig(8, dtype, root, 0, total / es, hash);
  const int blocks = vtable_grid(vt);
  rc = with_unit(st.in | st.out | vtable_bits(vt), [&](auto u) {
    return launch_coll(scatterv_pull_kernel<decltype(u), 4>, "scatterv_pull_kernel", sig, blocks, kThreads, 0, g->stream, st.in, st.out, vt, root);
  });
  return rc ? rc : finish(false, st);
}

// ReduceScatterv: one algorithm, the grid of the largest block.  UNROLL per element size is the
// largest power of two for which ptxas reports no spill in any instance.  The signature carries the
// total count and the table hash, so a rank with another table, op or dtype, or one calling
// ReduceScatter (code 4), ends the call as B200MPI_ERR_PEER on every rank.
static int launch_reduce_scatterv(int dtype, int op, uint64_t so, uint64_t ro, const VTable& vt, size_t es, uint64_t hash, cudaStream_t s) {
  const uint64_t sig = make_sig(13, dtype, op, 0, vt.off[g->ctrl.n] / es, hash);
  return with_reduction(
      dtype, op,
      [&](auto t, auto o) {
        using T = decltype(t);
        using Op = decltype(o);
        constexpr int U = sizeof(T) == 4 ? 8 : 4; // f64 min/max spilled at 8, every type at 16
        return launch_coll(reduce_scatterv_kernel<T, Op, U>, "reduce_scatterv_kernel", sig, vtable_grid(vt, U), kThreads, 0, s, so, ro, vt);
      },
      [] { return fail(B200MPI_ERR_UNSUPPORTED, "reduce_scatterv: unsupported dtype/op (need f32, f64 or i64 with sum/max/min)"); });
}

// ReduceScatterv: send holds sum(counts) elements; rank j's recv (counts[j] elements, NULL allowed
// when that is 0) receives op over r of block j of rank r's send.  In place: recv == send + the
// displacement of this rank's block.  Host slices and foreign device pointers are staged whole.
static int do_reduce_scatterv(const void* send, void* recv, const size_t* counts, int dtype, int op, int memkind) {
  size_t es;
  int rc = check_coll("reduce_scatterv", kReduces, dtype, op, 0, memkind, es);
  if (rc) return rc;
  const int n = g->ctrl.n, me = g->ctrl.rank;
  VTable vt;
  uint64_t hash;
  if ((rc = make_vtable("reduce_scatterv", counts, es, vt, hash))) return rc;
  const size_t mine = vt.off[me + 1] - vt.off[me], total = vt.off[n];
  if ((total && !send) || (mine && !recv)) return null_buffer("reduce_scatterv");
  if (n == 1) return local_copy(recv, send, mine, memkind, false); // counts[0] covers the whole send
  const bool inplace = recv && (const char*)recv == (const char*)send + vt.off[me];
  Staging st; // a NULL recv (counts[rank] == 0) announces the send offset and is never written
  if ((rc = stage(st, memkind, send, total, recv, mine, !recv ? kSendOnly : inplace ? kRecvInSend : kApart, vt.off[me]))) return rc;
  if ((rc = launch_reduce_scatterv(dtype, op, st.in, st.out, vt, es, hash, g->stream))) return rc;
  return finish(false, st);
}

// The fixed-count forms: the uniform table.
static int do_gather(const void* send, void* recv, size_t count, int dtype, int root, int memkind, bool scatter) {
  int rc = need_data_plane();
  if (rc) return rc;
  const std::vector<size_t> counts((size_t)g->ctrl.n, count);
  return scatter ? do_scatterv(send, recv, counts.data(), dtype, root, memkind) : do_gatherv(send, recv, counts.data(), dtype, root, false, memkind);
}

// Alltoallv: block j of send (send_counts[j] elements, packed in rank order) goes to rank j, where it
// lands at displacement recv_counts[0] + ... + recv_counts[rank()-1] of that rank's recv.  Every rank
// holds a different table, so the tables are checked on the device (sync_start_pairs) and a
// mismatch ends as B200MPI_ERR_PEER on every rank with no buffer touched.
static int do_alltoallv(const void* send, const size_t* send_counts, void* recv, const size_t* recv_counts, int dtype, int memkind) {
  size_t es;
  int rc = check_coll("alltoallv", 0, dtype, 0, 0, memkind, es);
  if (rc) return rc;
  const int n = g->ctrl.n, me = g->ctrl.rank;
  if (!send_counts || !recv_counts) return fail(B200MPI_ERR_ARG, "alltoallv: NULL counts table");
  VTable sv, rv;
  uint64_t digest;
  if (!a2av_tables(me, n, send_counts, recv_counts, es, sv, rv, digest)) return fail(B200MPI_ERR_ARG, "alltoallv: sum(counts) * element size overflows");
  const size_t sbytes = sv.off[n], rbytes = rv.off[n];
  if ((sbytes && !send) || (rbytes && !recv)) return null_buffer("alltoallv");
  if (send == recv && (sbytes || rbytes)) return fail(B200MPI_ERR_ARG, "alltoallv: in place is not supported");
  if (n == 1) {
    if (send_counts[0] != recv_counts[0]) return fail(B200MPI_ERR_PEER, "alltoallv: send_counts[0] != recv_counts[0] in a world of one; buffers were left untouched");
    return local_copy(recv, send, sbytes, memkind, false);
  }
  Staging st;
  if ((rc = stage(st, memkind, send, sbytes, recv, rbytes))) return rc;
  // The grid is block_cap() CTAs whatever the table: the barriers pair CTAs by blockIdx and the grid
  // is part of the signature, so it may depend only on what every rank shares.  The access unit
  // follows this rank's offsets and both of its displacement tables.  The table digest goes into the
  // signature this rank announces after the grid (sync_start_pairs), so this launch is its own.
  const int blocks = block_cap();
  Comm c = next_comm(make_sig(10, dtype, 0, 0, 0));
  sig_grid(c, blocks);
  const uint64_t base_sig = c.sig;
  c.sig = base_sig + digest;
  rc = with_unit(st.in | st.out | vtable_bits(sv) | vtable_bits(rv), [&](auto u) {
    alltoallv_push_kernel<decltype(u), 4><<<blocks, kThreads, 0, g->stream>>>(c, st.in, st.out, sv, rv, base_sig);
    return launch_check("alltoallv_push_kernel");
  });
  return rc ? rc : finish(false, st);
}

// ---------------------------------------------------------------------------------------------
// One-sided communication (active target, fence synchronisation).  A window is a range of each
// rank's heap whose offset and size every rank learns at win_create, so a Put, Get or Accumulate is
// one kernel between the origin (or its staging block) and base[target] + offset: not a collective,
// it takes no epoch.  Every RMA call is blocking, so at a fence this rank's RMA kernels have
// completed; the fence is then the barrier kernel under signature code 15 with the window id, whose
// release / acquire flags at system scope order those writes before every rank's later work.
// ---------------------------------------------------------------------------------------------
static Ctx::Win* find_win(int win) {
  return win >= 0 && (size_t)win < g->wins.size() && g->wins[win].live ? &g->wins[win] : nullptr;
}
static int unknown_win(const char* what) { return fail(B200MPI_ERR_ARG, std::string(what) + ": unknown or freed window"); }

// Collective.  Every rank announces {next id, heap offset, bytes, its own verdict on its arguments},
// so a rank with bad arguments fails with B200MPI_ERR_ARG and the others with B200MPI_ERR_PEER, and
// no rank creates the window.
static int do_win_create(void* base, size_t bytes, int* win) {
  int rc = need_data_plane();
  if (rc) return rc;
  size_t off = 0;
  const char* bad = nullptr;
  if (!win) bad = "NULL result pointer";
  else if ((base || bytes) && (!base || bytes > g->heap.size || !g->heap.contains(base, bytes, off)))
    bad = "window memory must lie in this rank's b200mpi_alloc heap (or be 0 bytes at NULL)";
  // The lowest free lock cell: create and free are collective and run in the same order on every rank,
  // so every rank picks the same one.  This rank zeroes its own cell (the lock word and the PSCW
  // counters) before the exchange, so no peer can lock it or signal into it before it is clear.
  g->lock_cell_used.resize(kWinLockCells);
  const uint64_t cell = std::find(g->lock_cell_used.begin(), g->lock_cell_used.end(), false) - g->lock_cell_used.begin();
  if (!bad && cell < kWinLockCells) {
    CUDA_OK(cudaMemsetAsync((char*)g->heap.base[g->ctrl.rank] + kWinLockOff + cell * kWinLockStride, 0, kWinLockStride, g->stream));
    CUDA_OK(cudaStreamSynchronize(g->stream));
  }
  struct { uint64_t id, off, bytes, bad, cell; } mine = {g->wins.size(), off, bytes, bad ? 1u : 0u, cell}, all[B200MPI_MAX_RANKS];
  std::string err;
  if ((rc = g->ctrl.allgather(&mine, sizeof mine, all, err, g->watchdog_ns > 0 ? g->watchdog_ns : -1))) return fail(rc, "win_create: " + err);
  if (bad) return fail(B200MPI_ERR_ARG, std::string("win_create: ") + bad);
  Ctx::Win w = {true, {}, {}, (uint32_t)cell, {}};
  for (int r = 0; r < g->ctrl.n; ++r) {
    if (all[r].bad) return fail(B200MPI_ERR_PEER, "win_create: rank " + std::to_string(r) + " refused its arguments");
    if (all[r].id != mine.id) return fail(B200MPI_ERR_PEER, "win_create: ranks disagree about the window id (" + std::to_string(all[r].id) + " on rank " + std::to_string(r) + ", " + std::to_string(mine.id) + " here)");
    if (all[r].cell != cell) return fail(B200MPI_ERR_PEER, "win_create: ranks disagree about the lock cell (" + std::to_string(all[r].cell) + " on rank " + std::to_string(r) + ", " + std::to_string(cell) + " here)");
    w.off[r] = all[r].off;
    w.bytes[r] = all[r].bytes;
  }
  if (cell >= kWinLockCells) return fail(B200MPI_ERR_NOMEM, "win_create: " + std::to_string(kWinLockCells) + " windows are live already");
  g->lock_cell_used[cell] = true;
  g->wins.push_back(w);
  *win = (int)mine.id;
  return 0;
}

// Collective: the barrier kernel under signature 15 carrying the window id, so a fence on another
// window or a Barrier ends as B200MPI_ERR_PEER on every rank.  A world of one synchronises the stream.
// free: the window is dropped once the fence has succeeded.  A rank that holds a lock on the window,
// or has an access or exposure epoch open on it, enters under a signature with the "locked" mark
// (extra = 1): the mismatch ends the call on every rank, as B200MPI_ERR_ARG here and
// B200MPI_ERR_PEER on the others, and the window, the lock and the epochs stay.
static int do_win_fence(int win, bool free) {
  const char* what = free ? "win_free" : "win_fence";
  int rc = need_data_plane();
  if (rc) return rc;
  Ctx::Win* w = find_win(win);
  if (!w) return unknown_win(what);
  const bool holds = std::any_of(w->held, w->held + B200MPI_MAX_RANKS, [](uint8_t h) { return h != 0; });
  const bool epoch = w->exposed || w->accessing;
  const bool locked = holds || epoch;
  const std::string held = std::string(what) + ": this rank " +
                           (holds && epoch ? "holds a lock on the window and has an access or exposure epoch open on it (unlock it, and complete or wait the epoch, first)"
                            : holds        ? "holds a lock on the window (unlock it first)"
                                           : "has an access or exposure epoch open on the window (complete or wait it first)");
  if (locked && g->ctrl.n == 1) return fail(B200MPI_ERR_ARG, held);
  if (g->ctrl.n > 1 && (rc = launch_coll(barrier_kernel, "barrier_kernel", make_sig(15, 0, locked ? 1 : 0, 0, (size_t)win), 1, 32, 0, g->stream))) return rc;
  rc = finish(false);
  if (locked) return fail(B200MPI_ERR_ARG, held); // also when every rank held one and the marks agreed
  if (rc) return rc;
  if (free) {
    w->live = false;
    g->lock_cell_used[w->lock_cell] = false;
  }
  return 0;
}

// with_reduction's dispatch for the one-sided calls, which also take REPLACE and NO_OP.
template <typename F, typename G>
static auto with_rma_op(int dtype, int op, F&& f, G&& otherwise) {
  auto more = [&] {
    auto g = [&](auto t) {
      if (op == B200MPI_REPLACE) return f(t, OpReplace{});
      if (op == B200MPI_NO_OP) return f(t, OpNoOp{});
      return otherwise();
    };
    switch (dtype) {
      case B200MPI_F32: return g(float{});
      case B200MPI_F64: return g(double{});
      case B200MPI_I64: return g(0ll);
    }
    return otherwise();
  };
  return with_reduction(dtype, op, f, more);
}

static int launch_accumulate(int dtype, int op, void* dst, const void* src, size_t count, cudaStream_t s) {
  auto unsupported = [] { return fail(B200MPI_ERR_UNSUPPORTED, "accumulate: unsupported dtype/op (need f32, f64 or i64 with sum/max/min/replace)"); };
  return with_rma_op(
      dtype, op,
      [&](auto t, auto o) {
        using T = decltype(t);
        if constexpr (std::is_same<decltype(o), OpNoOp>::value) {
          return unsupported();
        } else {
          accumulate_kernel<T, decltype(o)><<<copy_grid(count * sizeof(T)), 256, 0, s>>>((T*)dst, (const T*)src, count);
          return launch_check("accumulate_kernel");
        }
      },
      unsupported);
}

enum RmaKind { kPut, kGet, kAccumulate };

// `count` elements of `dtype` between origin and element target_disp of `target`'s window.  Blocking:
// returns once origin may be reused (Get: holds the data).  Host origins and device pointers outside
// the heap are staged whole, through block 0 (Put, Accumulate) or block 1 (Get).
static int do_rma(RmaKind kind, const void* origin, size_t count, int dtype, int op, int target, size_t target_disp, int win, int memkind) {
  static const char* const names[] = {"put", "get", "accumulate"};
  const char* what = names[kind];
  int rc = need_data_plane();
  if (rc) return rc;
  auto arg = [&](const char* msg) { return fail(B200MPI_ERR_ARG, std::string(what) + ": " + msg); };
  const Ctx::Win* w = find_win(win);
  if (!w) return unknown_win(what);
  const size_t es = esize(dtype);
  if (es == 0) return arg("unknown dtype");
  if (kind == kAccumulate && dtype == B200MPI_U8) return fail(B200MPI_ERR_UNSUPPORTED, "accumulate: dtype must be f32, f64 or i64");
  if (kind == kAccumulate && (op < B200MPI_SUM || op > B200MPI_REPLACE)) return arg("unknown op (accumulate takes sum, max, min or replace)");
  if (target < 0 || target >= g->ctrl.n) return arg("target out of range");
  if (memkind != B200MPI_HOST && memkind != B200MPI_DEVICE) return arg("bad memkind");
  if (count == 0) return 0;
  if (!origin) return arg("NULL origin with count > 0");
  // (target_disp + count) * es <= window bytes, without overflow
  if (target_disp > SIZE_MAX - count || target_disp + count > w->bytes[target] / es) return arg("target_disp + count elements exceed the target's window");
  const uint64_t at = w->off[target] + target_disp * es; // in the target's heap
  if (kind == kAccumulate && at % es) return arg("target element address is not a multiple of the element size");
  const size_t bytes = count * es;
  char* const remote = (char*)g->heap.base[target] + at;
  char* const local = (char*)g->heap.base[g->ctrl.rank];
  Buf b;
  if (kind == kGet) {
    if ((rc = resolve(origin, bytes, memkind, 1, false, b))) return rc;
    if ((rc = launch_copy(local + b.off, remote, bytes, g->stream))) return rc;
    return finish(false, Staging{0, b.off, b.staged ? const_cast<void*>(origin) : nullptr, bytes, memkind});
  }
  if ((rc = resolve(origin, bytes, memkind, 0, true, b))) return rc;
  if (kind == kPut) {
    rc = launch_copy(remote, local + b.off, bytes, g->stream);
  } else {
    if (b.off % es) { // a heap origin off its element alignment: the kernel loads whole elements
      if ((rc = ensure_stage(0, bytes))) return rc;
      b.off = g->stage_off[0];
      if ((rc = launch_local_copy(local + b.off, origin, bytes, g->stream))) return rc;
    }
    rc = launch_accumulate(dtype, op, remote, local + b.off, count, g->stream);
  }
  return rc ? rc : finish(false);
}

// ---------------------------------------------------------------------------------------------
// Passive target: window locks and the fetching atomics.  Not collectives, no epoch.  A lock is one
// 64-bit word per window in every rank's control region (kWinLockOff, kernels.cuh); win_lock relaunches
// win_lock_try_kernel, whose attempts are bounded, until it reports the lock or watchdog_ms has passed,
// so a waiting rank neither trips the device watchdog nor takes the collectives' resync path.  Every
// call ends in a stream synchronisation, so everything this rank did to a window before win_unlock has
// completed when the unlock kernel's release runs (DESIGN §3).
// ---------------------------------------------------------------------------------------------
static int need_rma_words() {
  if (g->rma_host) return 0;
  void* p = nullptr;
  if (cudaHostAlloc(&p, 64, cudaHostAllocMapped) != cudaSuccess) { (void)cudaGetLastError(); return fail(B200MPI_ERR_CUDA, "rma: mapped result words could not be allocated"); }
  if (cudaHostGetDevicePointer((void**)&g->rma_dev, p, 0) != cudaSuccess) { (void)cudaGetLastError(); cudaFreeHost(p); return fail(B200MPI_ERR_CUDA, "rma: mapped result words have no device address"); }
  g->rma_host = (uint64_t*)p;
  return 0;
}

static unsigned long long* lock_word(const Ctx::Win* w, int target) {
  return (unsigned long long*)((char*)g->heap.base[target] + kWinLockOff + (size_t)w->lock_cell * kWinLockStride);
}

static int do_win_lock(int lock_type, int target, int win) {
  int rc = need_data_plane();
  if (rc) return rc;
  Ctx::Win* w = find_win(win);
  if (!w) return unknown_win("win_lock");
  if (lock_type != B200MPI_LOCK_EXCLUSIVE && lock_type != B200MPI_LOCK_SHARED) return fail(B200MPI_ERR_ARG, "win_lock: lock type must be exclusive or shared");
  if (target < 0 || target >= g->ctrl.n) return fail(B200MPI_ERR_ARG, "win_lock: target out of range");
  if (w->held[target]) return fail(B200MPI_ERR_ARG, "win_lock: this rank already holds a lock on the target's window");
  if ((rc = need_rma_words())) return rc;
  volatile uint32_t* verdict = (volatile uint32_t*)(g->rma_host + 1);
  Spinner sp(g->watchdog_ns);
  for (;;) {
    *verdict = 2;
    win_lock_try_kernel<<<1, 1, 0, g->stream>>>(lock_word(w, target), lock_type == B200MPI_LOCK_EXCLUSIVE, (uint32_t*)(g->rma_dev + 1));
    if ((rc = launch_check("win_lock_try_kernel")) || (rc = finish(false))) return rc;
    if (*verdict == 1) break;
    if (sp.expired()) return fail(B200MPI_ERR_TIMEOUT, "win_lock: the lock was not granted within watchdog_ms");
  }
  w->held[target] = (uint8_t)lock_type;
  return 0;
}

static int do_win_unlock(int target, int win) {
  int rc = need_data_plane();
  if (rc) return rc;
  Ctx::Win* w = find_win(win);
  if (!w) return unknown_win("win_unlock");
  if (target < 0 || target >= g->ctrl.n) return fail(B200MPI_ERR_ARG, "win_unlock: target out of range");
  if (!w->held[target]) return fail(B200MPI_ERR_ARG, "win_unlock: this rank holds no lock on the target's window");
  win_unlock_kernel<<<1, 1, 0, g->stream>>>(lock_word(w, target), w->held[target] == B200MPI_LOCK_EXCLUSIVE);
  if ((rc = launch_check("win_unlock_kernel")) || (rc = finish(false))) return rc;
  w->held[target] = 0;
  return 0;
}

// The checks every fetching call makes first, in do_rma's order: the data plane, the window, the
// dtype, the op, the target; then (count > 0) the range and the element alignment of the target.
// `remote` is the target element through its peer mapping.  i64_only: compare_and_swap.
static int rma_atomic_target(const char* what, int dtype, int op, int target, size_t target_disp, size_t count, int win, char*& remote, bool i64_only = false) {
  int rc = need_data_plane();
  if (rc) return rc;
  auto arg = [&](const char* msg) { return fail(B200MPI_ERR_ARG, std::string(what) + ": " + msg); };
  const Ctx::Win* w = find_win(win);
  if (!w) return unknown_win(what);
  const size_t es = esize(dtype);
  if (es == 0) return arg("unknown dtype");
  if (dtype == B200MPI_U8 || (i64_only && dtype != B200MPI_I64)) return fail(B200MPI_ERR_UNSUPPORTED, std::string(what) + (i64_only ? ": dtype must be i64" : ": dtype must be f32, f64 or i64"));
  if (op < B200MPI_SUM || op > B200MPI_NO_OP) return arg("unknown op");
  if (target < 0 || target >= g->ctrl.n) return arg("target out of range");
  if (count == 0) return 0;
  if (target_disp > SIZE_MAX - count || target_disp + count > w->bytes[target] / es) return arg("target_disp + count elements exceed the target's window");
  const uint64_t at = w->off[target] + target_disp * es;
  if (at % es) return arg("target element address is not a multiple of the element size");
  remote = (char*)g->heap.base[target] + at;
  return 0;
}

// result[e] = target[e] before, target[e] = target[e] op origin[e].  Origin through staging block 0 and
// result through block 1 when they lie outside the heap or off their element alignment; result ==
// origin shares the origin's place.
static int do_get_accumulate(const void* origin, void* result, size_t count, int dtype, int op, int target, size_t target_disp, int win, int memkind) {
  const char* what = "get_accumulate";
  char* remote = nullptr;
  int rc = rma_atomic_target(what, dtype, op, target, target_disp, count, win, remote);
  if (rc) return rc;
  auto arg = [&](const char* msg) { return fail(B200MPI_ERR_ARG, std::string(what) + ": " + msg); };
  if (memkind != B200MPI_HOST && memkind != B200MPI_DEVICE) return arg("bad memkind");
  if (count == 0) return 0;
  const bool reads = op != B200MPI_NO_OP;
  if (reads && !origin) return arg("NULL origin with count > 0");
  if (!result) return arg("NULL result with count > 0");
  const size_t es = esize(dtype), bytes = count * es;
  const bool in_place = reads && result == origin;
  if (reads && !in_place && (uintptr_t)result < (uintptr_t)origin + bytes && (uintptr_t)origin < (uintptr_t)result + bytes)
    return arg("result overlaps origin without being it");
  char* const local = (char*)g->heap.base[g->ctrl.rank];
  Buf src, res;
  if (reads) {
    if ((rc = resolve(origin, bytes, memkind, 0, true, src))) return rc;
    if (src.off % es) { // a heap origin off its element alignment: the kernel loads whole elements
      if ((rc = ensure_stage(0, bytes))) return rc;
      src = {g->stage_off[0], true};
      if ((rc = launch_local_copy(local + src.off, origin, bytes, g->stream))) return rc;
    }
  }
  if (in_place) {
    res = src;
  } else {
    if ((rc = resolve(result, bytes, memkind, 1, false, res))) return rc;
    if (res.off % es) {
      if ((rc = ensure_stage(1, bytes))) return rc;
      res = {g->stage_off[1], true};
    }
  }
  rc = with_rma_op(
      dtype, op,
      [&](auto t, auto o) {
        using T = decltype(t);
        get_accumulate_kernel<T, decltype(o)><<<copy_grid(bytes), 256, 0, g->stream>>>((T*)remote, reads ? (const T*)(local + src.off) : nullptr, (T*)(local + res.off), count);
        return launch_check("get_accumulate_kernel");
      },
      [&] { return arg("unknown op"); });
  if (rc) return rc;
  return finish(false, Staging{0, res.off, res.staged ? result : nullptr, bytes, memkind});
}

// One element between host values: the operand as a kernel parameter, the old value through the
// mapped word.  One launch, no staging.
static int do_fetch_and_op(const void* origin, void* result, int dtype, int op, int target, size_t target_disp, int win) {
  const char* what = "fetch_and_op";
  char* remote = nullptr;
  int rc = rma_atomic_target(what, dtype, op, target, target_disp, 1, win, remote);
  if (rc) return rc;
  if (!origin && op != B200MPI_NO_OP) return fail(B200MPI_ERR_ARG, "fetch_and_op: NULL origin");
  if (!result) return fail(B200MPI_ERR_ARG, "fetch_and_op: NULL result");
  if ((rc = need_rma_words())) return rc;
  const size_t es = esize(dtype);
  rc = with_rma_op(
      dtype, op,
      [&](auto t, auto o) {
        using T = decltype(t);
        T v{};
        if (op != B200MPI_NO_OP) memcpy(&v, origin, sizeof(T));
        fetch_op_kernel<T, decltype(o)><<<1, 1, 0, g->stream>>>((T*)remote, v, (T*)g->rma_dev);
        return launch_check("fetch_op_kernel");
      },
      [] { return fail(B200MPI_ERR_ARG, "fetch_and_op: unknown op"); });
  if (rc || (rc = finish(false))) return rc;
  memcpy(result, (const void*)g->rma_host, es);
  return 0;
}

static int do_compare_and_swap(const void* origin, const void* compare, void* result, int dtype, int target, size_t target_disp, int win) {
  char* remote = nullptr;
  int rc = rma_atomic_target("compare_and_swap", dtype, B200MPI_REPLACE, target, target_disp, 1, win, remote, true);
  if (rc) return rc;
  if (!origin || !compare || !result) return fail(B200MPI_ERR_ARG, "compare_and_swap: NULL origin, compare or result");
  if ((rc = need_rma_words())) return rc;
  unsigned long long v, c;
  memcpy(&v, origin, 8);
  memcpy(&c, compare, 8);
  cas_kernel<<<1, 1, 0, g->stream>>>((unsigned long long*)remote, c, v, (unsigned long long*)g->rma_dev);
  if ((rc = launch_check("cas_kernel")) || (rc = finish(false))) return rc;
  memcpy(result, (const void*)g->rma_host, 8);
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Generalized active target: post / start / complete / wait / test.  Not collectives, no epoch, and
// only the ranks named in a group take part.  Each pair of ranks counts its epochs on the window in
// two 16-bit words of the window's cell (kPscwPostedOff, kPscwCompletedOff in kernels.cuh): post and
// complete store the new count into the peer's cell (pscw_signal_kernel), start and wait poll this
// rank's own cell for the count they expect (pscw_poll_kernel, relaunched for the members still
// missing until all have arrived or watchdog_ms has passed).  Every call ends in a stream
// synchronisation, which is the ordering argument of win_unlock (DESIGN §3).
// ---------------------------------------------------------------------------------------------
static uint16_t* pscw_word(const Ctx::Win* w, int owner, size_t off, int peer) {
  return (uint16_t*)((char*)g->heap.base[owner] + kWinLockOff + (size_t)w->lock_cell * kWinLockStride + off) + peer;
}

// `count` distinct ranks in [0, size()) as a mask; nullptr when well formed, else what is wrong.
static const char* pscw_group(const int* ranks, int count, uint8_t& mask) {
  mask = 0;
  if (count < 0) return "negative group size";
  if (count > g->ctrl.n) return "group larger than the world";
  if (count > 0 && !ranks) return "NULL group with count > 0";
  for (int i = 0; i < count; ++i) {
    if (ranks[i] < 0 || ranks[i] >= g->ctrl.n) return "rank in the group out of range";
    if (mask >> ranks[i] & 1) return "rank repeated in the group";
    mask |= (uint8_t)(1u << ranks[i]);
  }
  return nullptr;
}

// Stores count[r] into the word `off` of every member r's cell at index this rank: one launch, none
// for an empty group.
static int pscw_signal(const Ctx::Win* w, uint8_t mask, size_t off, const uint16_t* count) {
  PscwGroup grp{};
  int m = 0;
  for (int r = 0; r < g->ctrl.n; ++r)
    if (mask >> r & 1) {
      grp.word[m] = pscw_word(w, r, off, g->ctrl.rank);
      grp.count[m++] = count[r];
    }
  if (m == 0) return 0;
  pscw_signal_kernel<<<1, m, 0, g->stream>>>(grp);
  const int rc = launch_check("pscw_signal_kernel");
  return rc ? rc : finish(false);
}

// Polls the words `off` of this rank's cell at the members of `mask` until each holds want[r]: one
// launch per pass, the next pass for the members still missing, a single pass of one attempt for
// `once` (win_test).  `all`: every member arrived.  An empty group launches nothing.
static int pscw_poll(const Ctx::Win* w, uint8_t mask, size_t off, const uint16_t* want, bool once, bool& all) {
  int rc = need_rma_words();
  if (rc) return rc;
  volatile uint8_t* arrived = (volatile uint8_t*)(g->rma_host + 2);
  Spinner sp(g->watchdog_ns);
  uint8_t missing = mask;
  while (missing) {
    PscwGroup grp{};
    int ranks[B200MPI_MAX_RANKS], m = 0;
    for (int r = 0; r < g->ctrl.n; ++r)
      if (missing >> r & 1) {
        grp.word[m] = pscw_word(w, g->ctrl.rank, off, r);
        grp.count[m] = want[r];
        ranks[m++] = r;
      }
    for (int i = 0; i < m; ++i) arrived[i] = 2;
    pscw_poll_kernel<<<1, m, 0, g->stream>>>(grp, once ? 1 : kPscwAttempts, (uint8_t*)(g->rma_dev + 2));
    if ((rc = launch_check("pscw_poll_kernel")) || (rc = finish(false))) return rc;
    for (int i = 0; i < m; ++i)
      if (arrived[i] == 1) missing &= (uint8_t)~(1u << ranks[i]);
    if (once || sp.expired()) break;
  }
  all = missing == 0;
  return 0;
}

// The checks every PSCW call makes first, in this order: the data plane, the window, then (post and
// start) the group.
static int pscw_checks(const char* what, int win, Ctx::Win*& w, const int* ranks = nullptr, int count = 0, uint8_t* mask = nullptr) {
  int rc = need_data_plane();
  if (rc) return rc;
  if (!(w = find_win(win))) return unknown_win(what);
  if (mask)
    if (const char* bad = pscw_group(ranks, count, *mask)) return fail(B200MPI_ERR_ARG, std::string(what) + ": " + bad);
  return 0;
}

// Opens an exposure epoch to `origins`: their posted[this rank] words take the epoch's count.
static int do_win_post(const int* origins, int count, int win) {
  Ctx::Win* w = nullptr;
  uint8_t mask = 0;
  int rc = pscw_checks("win_post", win, w, origins, count, &mask);
  if (rc) return rc;
  if (w->exposed) return fail(B200MPI_ERR_ARG, "win_post: this rank's exposure epoch on the window is open already (win_wait closes it)");
  uint16_t next[B200MPI_MAX_RANKS];
  for (int r = 0; r < B200MPI_MAX_RANKS; ++r) next[r] = (uint16_t)(w->exposures[r] + 1);
  if ((rc = pscw_signal(w, mask, kPscwPostedOff, next))) return rc;
  for (int r = 0; r < g->ctrl.n; ++r)
    if (mask >> r & 1) w->exposures[r] = next[r];
  w->exposed = true;
  w->expose_group = mask;
  return 0;
}

// Opens an access epoch to `targets` once each has posted to this rank: posted[t] reaches the count
// of this start.  On a timeout nothing changes, so a post that did arrive is seen by the next start.
static int do_win_start(const int* targets, int count, int win) {
  Ctx::Win* w = nullptr;
  uint8_t mask = 0;
  int rc = pscw_checks("win_start", win, w, targets, count, &mask);
  if (rc) return rc;
  if (w->accessing) return fail(B200MPI_ERR_ARG, "win_start: this rank's access epoch on the window is open already (win_complete closes it)");
  uint16_t next[B200MPI_MAX_RANKS];
  for (int r = 0; r < B200MPI_MAX_RANKS; ++r) next[r] = (uint16_t)(w->accesses[r] + 1);
  bool all = false;
  if ((rc = pscw_poll(w, mask, kPscwPostedOff, next, false, all))) return rc;
  if (!all) return fail(B200MPI_ERR_TIMEOUT, "win_start: a target did not post to this rank within watchdog_ms; no access epoch is open");
  for (int r = 0; r < g->ctrl.n; ++r)
    if (mask >> r & 1) w->accesses[r] = next[r];
  w->accessing = true;
  w->access_group = mask;
  return 0;
}

// Closes the access epoch: every target's completed[this rank] word takes the epoch's count.
static int do_win_complete(int win) {
  Ctx::Win* w = nullptr;
  int rc = pscw_checks("win_complete", win, w);
  if (rc) return rc;
  if (!w->accessing) return fail(B200MPI_ERR_ARG, "win_complete: this rank has no access epoch open on the window");
  if ((rc = pscw_signal(w, w->access_group, kPscwCompletedOff, w->accesses))) return rc;
  w->accessing = false;
  w->access_group = 0;
  return 0;
}

// Closes the exposure epoch once every origin has completed: completed[o] reaches the count of the
// post.  win_wait (flag == nullptr) waits up to watchdog_ms; win_test looks once.  Either way an epoch
// that has not ended stays open.
static int do_win_wait(int win, int* flag, bool test) {
  const char* what = test ? "win_test" : "win_wait";
  Ctx::Win* w = nullptr;
  int rc = pscw_checks(what, win, w);
  if (rc) return rc;
  if (test && !flag) return fail(B200MPI_ERR_ARG, "win_test: NULL flag");
  if (!w->exposed) return fail(B200MPI_ERR_ARG, std::string(what) + ": this rank has no exposure epoch open on the window");
  bool all = false;
  if ((rc = pscw_poll(w, w->expose_group, kPscwCompletedOff, w->exposures, test, all))) return rc;
  if (test) *flag = all ? 1 : 0;
  if (!all) return test ? 0 : fail(B200MPI_ERR_TIMEOUT, "win_wait: an origin did not complete within watchdog_ms; the exposure epoch stays open");
  w->exposed = false;
  w->expose_group = 0;
  return 0;
}

// ---------------------------------------------------------------------------------------------
// point to point
// ---------------------------------------------------------------------------------------------
static Ctx::P2PBounce* acquire_bounce() {
  std::lock_guard<std::mutex> l(g->p2p_mu);
  for (auto& b : g->p2p_bounce) {
    if (b.busy) continue;
    if (!b.host) {
      void* p = nullptr;
      const size_t len = Ctx::kP2PBounceBytes + 64;
      cudaError_t e = on_numa_node(g->gpu_numa_node, [&] { return cudaHostAlloc(&p, len, cudaHostAllocMapped); });
      if (e != cudaSuccess || cudaHostGetDevicePointer((void**)&b.dev, p, 0) != cudaSuccess) { (void)cudaGetLastError(); if (p) cudaFreeHost(p); return nullptr; }
      b.host = (char*)p;
      *(volatile uint32_t*)(b.host + Ctx::kP2PBounceBytes) = 0;
    }
    b.busy = true;
    return &b;
  }
  return nullptr;
}
static void release_bounce(Ctx::P2PBounce* b) {
  std::lock_guard<std::mutex> l(g->p2p_mu);
  b->busy = false;
}
// dst <- src with the copy kernel on `s`, then spin on the bounce's completion word.  One of dst / src
// is the bounce's device mapping.  0, or an error (watchdog / launch failure).
static int copy_and_wait(Ctx::P2PBounce* b, void* dst, const void* src, size_t bytes, cudaStream_t s) {
  int rc = launch_copy(dst, src, bytes, s);
  if (rc) return rc;
  const uint32_t seq = ++b->seq;
  flag_kernel<<<1, 1, 0, s>>>((uint32_t*)(b->dev + Ctx::kP2PBounceBytes), seq);
  if ((rc = launch_check("flag_kernel"))) return rc;
  volatile uint32_t* done = (volatile uint32_t*)(b->host + Ctx::kP2PBounceBytes);
  Spinner sp(g->watchdog_ns);
  while (*done != seq)
    if (!sp.step()) { cudaStreamSynchronize(s); return fail(B200MPI_ERR_TIMEOUT, "p2p: copy kernel did not complete"); }
  std::atomic_thread_fence(std::memory_order_acquire);
  return 0;
}

static size_t p2p_chunk(size_t bytes, int memkind) {
  // Host slices: small chunks so the sender's H2D of chunk k+1 overlaps the receiver's pull + D2H of
  // chunk k (both block their host thread for pageable memory).  Device buffers: one big chunk.
  if (memkind == B200MPI_HOST) return std::min(g->stage_chunk, std::max<size_t>(64u << 10, (bytes / 4 + 4095) / 4096 * 4096));
  return g->stage_chunk;
}

static MsgSlot* claim_slot(int dest) {
  const int me = g->ctrl.rank;
  Spinner sp(g->watchdog_ns);
  for (;;) {
    for (int k = 0; k < kSlotsPerPair; ++k) {
      uint32_t expect = kFree;
      MsgSlot* s = &g->box->slots[me][dest][k];
      if (s->state.compare_exchange_strong(expect, kClaimed, std::memory_order_acq_rel)) return s;
    }
    if (!sp.step()) return nullptr;
  }
}

// The message could not be delivered (timeout / staging error).  Withdraw the post if nobody
// matched it; if a receiver is in the middle of pulling, the staging block must outlive it.
// Returns true when the slot and the staging block may be reused.
static bool retire_failed_send(MsgSlot* slot) {
  uint32_t expect = kPosted;
  if (slot->state.compare_exchange_strong(expect, kFree, std::memory_order_acq_rel)) return true;
  if (expect == kClaimed) { slot->state.store(kFree, std::memory_order_release); return true; }
  Spinner sp(g->watchdog_ns);
  while (slot->state.load(std::memory_order_acquire) != kDone)
    if (!sp.step()) return false; // receiver is stuck mid-pull: leak slot and staging rather than free memory it reads
  slot->state.store(kFree, std::memory_order_release);
  return true;
}

struct PendingSend { MsgSlot* slot; size_t stage; bool staged; };
static std::mutex g_pending_mu;
static std::map<std::pair<int, int>, PendingSend> g_pending; // {dest, tag} -> posted, not yet acknowledged (Isend)

// What Send, Isend and Receive check first, in this order: the data plane, the dtype, the peer, the
// buffer and the memory kind.  what is "send" or "recv"; es receives the element size.
static int check_p2p(const char* what, int dtype, int peer, const void* buf, size_t count, int memkind, size_t& es) {
  int rc = need_data_plane();
  if (rc) return rc;
  const bool send = !strcmp(what, "send");
  auto arg = [&](const std::string& msg) { return fail(B200MPI_ERR_ARG, std::string(what) + ": " + msg); };
  es = esize(dtype);
  if (es == 0) return arg("unknown dtype");
  if (peer < 0 || peer >= g->ctrl.n) return arg((send ? "destination " : "source ") + std::to_string(peer) + " out of range");
  if (count && !buf) return arg(send ? "NULL buffer with count > 0" : "NULL buffer with capacity > 0");
  if (memkind != B200MPI_HOST && memkind != B200MPI_DEVICE) return arg("bad memkind");
  return 0;
}

// Gives a {peer, tag} taken in `tags` back when the call that took it returns, unless an Isend
// hands it on to b200mpi_wait (keep).
struct TagRelease {
  TagSet& tags;
  int tag;
  bool keep = false;
  ~TagRelease() { if (!keep) tags.remove(tag); }
};

// The end of a Send, or of an Isend in b200mpi_wait: wait for the receiver's acknowledgement
// (network.go:569), then free the staging block and the slot.  After a failure (rc != 0, or no
// acknowledgement within the watchdog time) the post is withdrawn and the failure's message kept.
static int finish_send(const char* what, const PendingSend& ps, int rc) {
  if (rc == 0) {
    Spinner sp(g->watchdog_ns);
    while (ps.slot->state.load(std::memory_order_acquire) != kDone)
      if (!sp.step()) { rc = fail(B200MPI_ERR_TIMEOUT, std::string(what) + ": no matching receive within the watchdog time"); break; }
  }
  if (rc == 0) {
    if (ps.staged) g->heap.free_off(ps.stage);
    ps.slot->state.store(kFree, std::memory_order_release);
  } else {
    const std::string why = t_err;
    if (retire_failed_send(ps.slot) && ps.staged) g->heap.free_off(ps.stage);
    t_err = why;
  }
  return rc;
}

// wait_ack = true: mpi.Send (network.go:518-572), returns after the receiver's acknowledgement.
// wait_ack = false: the Send of the design sketched in mpi.go:132-152 -- returns once the data has
// left the caller's buffer ("sent on connection"); b200mpi_wait collects the acknowledgement.
static int do_send(const void* buf, size_t count, int dtype, int dest, int tag, int memkind, bool wait_ack) {
  size_t es;
  int rc = check_p2p("send", dtype, dest, buf, count, memkind, es);
  if (rc) return rc;
  if (!g->sendtags[dest].add(tag)) return fail(B200MPI_ERR_TAG_EXISTS, "Tag " + std::to_string(tag) + " already in use sending"); // mpi.go:180-182
  TagRelease held{g->sendtags[dest], tag};
  MsgSlot* slot = claim_slot(dest);
  if (!slot) return fail(B200MPI_ERR_TIMEOUT, "send: no free mailbox slot");
  const size_t bytes = count * es;
  // The layout.  Direct: the receiver pulls straight out of the caller's heap buffer (a Send only;
  // an Isend leaves the caller's buffer free).  Staged whole: an Isend keeps the whole message in the
  // staging block until Wait, and a small host slice goes through a mapped pinned bounce, where one
  // kernel moves it into the heap (the SMs read host memory over PCIe).  Otherwise a Send streams the
  // message through a ring of up to kMsgRegions chunks.
  PendingSend ps{slot, 0, false};
  size_t off = 0;
  const bool direct = bytes == 0 || (wait_ack && memkind == B200MPI_DEVICE && g->heap.contains(buf, bytes, off));
  Ctx::P2PBounce* bounce = !direct && memkind == B200MPI_HOST && g->p2p_fast && bytes <= Ctx::kP2PBounceBytes ? acquire_bounce() : nullptr;
  const size_t chunk = direct || bounce || !wait_ack ? bytes : std::min(bytes, p2p_chunk(bytes, memkind));
  const size_t nchunks = direct ? 0 : (bytes + chunk - 1) / chunk;
  const size_t nreg = std::min<size_t>(std::max<size_t>(nchunks, 1), kMsgRegions);
  if (!direct) {
    if (g->heap.alloc(chunk * nreg, ps.stage)) rc = fail(B200MPI_ERR_NOMEM, "send: symmetric heap exhausted while staging (raise B200MPI_HEAP_BYTES)");
    else ps.staged = true;
  }
  if (rc == 0) {
    slot->tag = tag;
    slot->dtype = (uint32_t)dtype;
    slot->result = 0;
    slot->count = count;
    slot->total_bytes = bytes;
    slot->chunk_bytes = chunk;
    slot->nregions = (uint32_t)nreg;
    for (size_t r = 0; r < nreg; ++r) slot->region_off[r] = direct ? off : ps.stage + r * chunk;
    slot->done.store(0, std::memory_order_relaxed);
    slot->posted.store(direct ? bytes : 0, std::memory_order_relaxed);
    slot->state.store(kPosted, std::memory_order_release);
  }
  // The fill: each chunk moves into its region and is then published in `posted`.
  cudaStream_t s = rc == 0 && nchunks ? borrow_stream() : nullptr;
  char* base = (char*)g->heap.base[g->ctrl.rank];
  for (size_t k = 0; k < nchunks && rc == 0; ++k) {
    if (k >= nreg) { // the region was used by chunk k-nreg: wait until the receiver drained it
      Spinner sp(g->watchdog_ns);
      while (slot->done.load(std::memory_order_acquire) < (k - nreg + 1) * chunk && slot->state.load(std::memory_order_acquire) != kDone)
        if (!sp.step()) { rc = fail(B200MPI_ERR_TIMEOUT, "send: receiver stalled"); break; }
      if (rc) break;
    }
    if (slot->state.load(std::memory_order_acquire) == kDone) break; // the receiver gave up (dtype mismatch or failure)
    const size_t lo = k * chunk, len = std::min(chunk, bytes - lo);
    char* to = base + slot->region_off[k % nreg];
    const char* from = (const char*)buf + lo;
    if (bounce) {
      memcpy(bounce->host, from, len);
      rc = copy_and_wait(bounce, to, bounce->dev, len, s);
    } else {
      cudaError_t e = cudaSuccess;
      if (memkind == B200MPI_HOST) e = cudaMemcpyAsync(to, from, len, cudaMemcpyHostToDevice, s);
      else rc = launch_copy(to, from, len, s);
      if (e == cudaSuccess && rc == 0) e = cudaStreamSynchronize(s);
      if (e != cudaSuccess) rc = fail(B200MPI_ERR_CUDA, std::string("send staging: ") + cudaGetErrorString(e));
    }
    if (rc == 0) slot->posted.store(lo + len, std::memory_order_release);
  }
  if (bounce) release_bounce(bounce);
  if (s) return_stream(s);
  if (rc == 0 && !wait_ack) { // Isend: the acknowledgement is collected by b200mpi_wait
    std::lock_guard<std::mutex> l(g_pending_mu);
    g_pending[{dest, tag}] = ps;
    held.keep = true;
    return 0;
  }
  return finish_send("send", ps, rc);
}

// mpi.go:146-152 (commented design): block until `destination` confirmed the message sent with
// `tag`, then free the {destination, tag} pair.
static int do_wait(int dest, int tag) {
  int rc = need_data_plane();
  if (rc) return rc;
  PendingSend ps;
  {
    std::lock_guard<std::mutex> l(g_pending_mu);
    auto it = g_pending.find({dest, tag});
    if (it == g_pending.end()) return fail(B200MPI_ERR_ARG, "wait: no unacknowledged send to " + std::to_string(dest) + " with tag " + std::to_string(tag));
    ps = it->second;
    g_pending.erase(it);
  }
  TagRelease held{g->sendtags[dest], tag};
  return finish_send("wait", ps, 0);
}

static int do_recv(void* buf, size_t capacity, size_t* count_out, int dtype, int src, int tag, int memkind) {
  size_t es;
  int rc = check_p2p("recv", dtype, src, buf, capacity, memkind, es);
  if (rc) return rc;
  if (!g->recvtags[src].add(tag)) return fail(B200MPI_ERR_TAG_EXISTS, "Tag " + std::to_string(tag) + " already in use receiving");
  TagRelease held{g->recvtags[src], tag};
  const int me = g->ctrl.rank;
  MsgSlot* slot = nullptr;
  {
    Spinner sp(g->watchdog_ns);
    for (;;) {
      for (int k = 0; k < kSlotsPerPair && !slot; ++k) {
        MsgSlot* s = &g->box->slots[src][me][k];
        if (s->state.load(std::memory_order_acquire) == kPosted && s->tag == tag) {
          uint32_t expect = kPosted;
          if (s->state.compare_exchange_strong(expect, kMatched, std::memory_order_acq_rel)) {
            if (s->tag == tag) slot = s;
            else s->state.store(kPosted, std::memory_order_release); // the slot was recycled between the look and the CAS
          }
        }
      }
      if (slot) break;
      if (!sp.step()) return fail(B200MPI_ERR_TIMEOUT, "recv: no matching send within the watchdog time");
    }
  }
  const size_t count = slot->count, bytes = slot->total_bytes;
  if (count_out) *count_out = count;
  if (slot->dtype != (uint32_t)dtype) {
    rc = fail(B200MPI_ERR_ARG, "recv: sender used dtype " + std::to_string(slot->dtype) + ", receiver asked for " + std::to_string(dtype));
  } else if (count > capacity) {
    // Nothing is consumed: the message stays posted so the caller can retry with a buffer of
    // *count_out elements (what gob's slice resize does for the reference, network.go:597).
    slot->state.store(kPosted, std::memory_order_release);
    return fail(B200MPI_ERR_TRUNCATE, "recv: message has " + std::to_string(count) + " elements, capacity is " + std::to_string(capacity));
  }
  // The pull unit.  A small message into a host slice, when every chunk has its own region (so the
  // message lies contiguous in the sender's heap), is pulled whole once all of it is posted: ONE
  // kernel moves it over NVLink straight into a mapped pinned bounce (the SMs write host memory),
  // then a memcpy.  Otherwise each chunk is pulled as soon as it is posted, into a device buffer
  // directly, or through a staging block and a D2H copy into a host slice.  That staging block is
  // at most this rank's stage_chunk, whatever the sender's layout: a chunk larger than that (a direct
  // post or an Isend is one chunk of the whole message) is pulled in several units, so that the heap a
  // host receive needs does not depend on the memory the sender passed.
  const size_t nreg = slot->nregions ? slot->nregions : 1, chunk = slot->chunk_bytes;
  Ctx::P2PBounce* bounce = nullptr;
  if (rc == 0 && bytes && memkind == B200MPI_HOST && g->p2p_fast && chunk * nreg >= bytes && bytes <= Ctx::kP2PBounceBytes) bounce = acquire_bounce();
  const size_t unit = bounce ? bytes : memkind == B200MPI_HOST ? std::min(chunk, g->stage_chunk) : chunk;
  size_t stage = 0;
  const bool staged = rc == 0 && bytes && !bounce && memkind == B200MPI_HOST;
  if (staged && g->heap.alloc(unit, stage)) {
    // Nothing is consumed, as for a truncation: the message stays posted, so the caller can free heap
    // memory and receive it again.
    slot->state.store(kPosted, std::memory_order_release);
    return fail(B200MPI_ERR_NOMEM, "recv: symmetric heap exhausted while staging " + std::to_string(unit) + " bytes (raise B200MPI_HEAP_BYTES or lower stage_chunk)");
  }
  cudaStream_t s = rc == 0 && bytes ? borrow_stream() : nullptr;
  const char* peer = (const char*)g->heap.base[src];
  char* mine = (char*)g->heap.base[me];
  for (size_t lo = 0, len = 0; rc == 0 && lo < bytes; lo += len) {
    // The sender publishes `posted` only at the end of a chunk, and reuses a region once `done` has
    // passed the end of its chunk: a unit never crosses a chunk's end (the bounce's one unit is the
    // whole message, contiguous in the sender's heap).
    len = bounce ? bytes : std::min({unit, chunk - lo % chunk, bytes - lo});
    Spinner sp(g->watchdog_ns);
    while (slot->posted.load(std::memory_order_acquire) < lo + len)
      if (!sp.step()) { rc = fail(B200MPI_ERR_TIMEOUT, "recv: sender stalled"); break; }
    if (rc) break;
    const char* from = peer + slot->region_off[lo / chunk % nreg] + lo % chunk;
    cudaError_t e = cudaSuccess;
    if (bounce) {
      rc = copy_and_wait(bounce, bounce->dev, from, len, s);
      if (rc == 0) memcpy((char*)buf + lo, bounce->host, len);
    } else {
      rc = launch_copy(memkind == B200MPI_DEVICE ? (char*)buf + lo : mine + stage, from, len, s);
      if (rc == 0 && memkind == B200MPI_HOST) e = cudaMemcpyAsync((char*)buf + lo, mine + stage, len, cudaMemcpyDeviceToHost, s);
      if (rc == 0 && e == cudaSuccess) e = cudaStreamSynchronize(s);
    }
    if (rc == 0 && e != cudaSuccess) rc = fail(B200MPI_ERR_CUDA, std::string("recv pull: ") + cudaGetErrorString(e));
    if (rc == 0) slot->done.store(lo + len, std::memory_order_release);
  }
  if (bounce) release_bounce(bounce);
  if (s) return_stream(s);
  if (staged) g->heap.free_off(stage);
  slot->result = rc;
  slot->state.store(kDone, std::memory_order_release); // the ack (network.go:617-621)
  return rc;
}

} // namespace b200

// =============================================================================================
// C ABI
// =============================================================================================
using namespace b200;

extern "C" {

int b200mpi_version(void) { return B200MPI_VERSION; }
const char* b200mpi_last_error(void) { return t_err.c_str(); }
int b200mpi_rank(void) { return (g && g->initialised) ? g->ctrl.rank : -1; }
int b200mpi_size(void) { return (g && g->initialised) ? g->ctrl.n : 0; }
int b200mpi_device(void) { return (g && g->initialised && !g->control_only) ? g->dev : -1; }
int64_t b200mpi_launch_count(void) { return g ? g->launches.load() : 0; }

// The tuning knobs of set_param / get_param, one row each; sm_count and the rows after it are read only.
// The compiled-in defaults are the member initialisers of Ctx.
using KnobField = std::variant<bool Ctx::*, int Ctx::*, uint32_t Ctx::*, int64_t Ctx::*, size_t Ctx::*>;
constexpr int64_t kLaneCap = -1; // as hi: the world's LL lane capacity, ll_cells(n) * 8 (ll_max_bytes only)
struct Knob {
  const char* name;
  KnobField field;                                   // holds value * scale (a bool holds value != 0)
  const char* env = nullptr;                         // B200MPI_* variable that overrides the default at Init
  int64_t lo = INT64_MIN, hi = INT64_MAX, scale = 1; // clamp, in set_param's units
};
static const Knob kKnobs[] = {
    {"twoshot_unroll", &Ctx::twoshot_unroll},
    {"nvls_unroll", &Ctx::nvls_unroll},
    {"nvls_min_ranks", &Ctx::nvls_min_ranks},
    {"nvls_max_blocks", &Ctx::nvls_max_blocks, nullptr, 1},
    {"oneshot_max_bytes", &Ctx::oneshot_max_bytes, "B200MPI_ONESHOT_MAX"},
    {"ll_max_bytes", &Ctx::ll_max_bytes, "B200MPI_LL_MAX", 0, kLaneCap},
    {"stage_chunk", &Ctx::stage_chunk, "B200MPI_STAGE_CHUNK", 4096},
    {"pipe_min_bytes", &Ctx::pipe_min_bytes},
    {"pipe_chunk_bytes", &Ctx::pipe_chunk_bytes, nullptr, 65536},
    {"bounce_chunk_bytes", &Ctx::bounce_chunk_bytes, nullptr, 65536},
    {"host_threads", &Ctx::host_threads, "B200MPI_HOST_THREADS", 0},
    {"own_block_bytes", &Ctx::own_block_bytes, nullptr, 4096},
    {"hybrid_p2p_permille", &Ctx::hybrid_p2p_permille, "B200MPI_HYBRID_PERMILLE", 0, 900},
    {"hybrid_p2p_blocks", &Ctx::hybrid_p2p_blocks, nullptr, 0},
    {"hybrid_min_bytes", &Ctx::hybrid_min_bytes, nullptr, 0},
    {"bcast_nvls2", &Ctx::bcast_nvls2},
    {"bcast_nvls_min", &Ctx::bcast_nvls_min, nullptr, 0},
    {"allgather_nvls_min", &Ctx::allgather_nvls_min, nullptr, 0},
    {"host_register", &Ctx::host_register, "B200MPI_HOST_REGISTER"},
    {"p2p_fast", &Ctx::p2p_fast, "B200MPI_P2P_FAST"},
    {"watchdog_ms", &Ctx::watchdog_ns, nullptr, 1, INT64_MAX, 1000000},
    {"sm_count", &Ctx::sm_count},
    {"shared_device", &Ctx::shared_device},
    {"epoch", &Ctx::epoch},
    {"ll_seq", &Ctx::ll_seq},
};
static const Knob* find_knob(const char* name) {
  for (const Knob& k : kKnobs) if (name && strcmp(name, k.name) == 0) return &k;
  return nullptr;
}
// The one clamp of a knob, for set_param and the environment alike: the row's range, then what the field
// holds, scaled.  A size_t field takes a negative value as its bit pattern, which get_param gives back.
static void store_knob(const Knob& k, int64_t v) {
  v = std::max(k.lo, std::min(v, k.hi == kLaneCap ? (int64_t)(ll_cells(g->ctrl.n) * 8) : k.hi));
  std::visit([&](auto m) {
    using T = std::remove_reference_t<decltype(g->*m)>;
    constexpr bool narrow = sizeof(T) < sizeof(int64_t);
    const int64_t tlo = narrow ? (int64_t)std::numeric_limits<T>::min() : INT64_MIN;
    const int64_t thi = narrow ? (int64_t)std::numeric_limits<T>::max() : INT64_MAX;
    if constexpr (std::is_same_v<T, bool>) g->*m = v != 0;
    else g->*m = (T)(std::clamp(v, tlo / k.scale, thi / k.scale) * k.scale);
  }, k.field);
}
// Init's last word on the knobs.  First the defaults that follow from the world: functions of n and
// of shared_device only, so every rank agrees.  Then every B200MPI_* override, through the clamp.
static void settle_knobs() {
  if (!g->control_only) {
    // LL (no barrier, one exchange latency) over its whole range on real multi-GPU worlds
    if (!g->shared_device) g->ll_max_bytes = std::min<size_t>(256u << 10, ll_cells(g->ctrl.n) * 8);
    // ranks time-slicing one GPU (functional-test mode): every extra kernel costs a time slice, keep the
    // host-slice Send/Receive on the copy-engine path there
    g->p2p_fast = !g->shared_device;
  }
  for (const Knob& k : kKnobs)
    if (const char* w = k.env ? getenv(k.env) : nullptr) store_knob(k, strtoll(w, nullptr, 0));
}
// Unregisters the host_register cache after the copies that may use it; no CUDA call when it is empty.
static void drop_registrations() {
  if (g->registered.empty()) return;
  cudaStreamSynchronize(g->h2d_stream);
  cudaStreamSynchronize(g->d2h_stream);
  for (auto& e : g->registered) cudaHostUnregister((void*)e.first);
  g->registered.clear();
  (void)cudaGetLastError();
}
// Releases everything a Ctx owns and deletes it, each release guarded, so it also undoes a partial Init.
static void teardown() {
  drop_registrations(); // while the copy streams it synchronises still exist
  for (cudaStream_t s : g->stream_pool) cudaStreamDestroy(s);
  for (cudaStream_t s : {g->own_stream, g->h2d_stream, g->d2h_stream}) if (s) cudaStreamDestroy(s);
  for (cudaEvent_t e : g->pipe_events) cudaEventDestroy(e);
  for (cudaEvent_t e : {g->ev0, g->ev1}) if (e) cudaEventDestroy(e);
  if (g->pool.running()) g->pool.shutdown(); // its threads fill the bounce ring
  for (void* p : {(void*)g->bounce, (void*)g->status_host, (void*)g->ll_host, (void*)g->rma_host}) if (p) cudaFreeHost(p);
  for (auto& b : g->p2p_bounce) if (b.host) cudaFreeHost(b.host);
  if (g->box) munmap(g->box, sizeof(Mailbox));
  {
    std::lock_guard<std::mutex> l(g_pending_mu);
    g_pending.clear();
  }
  g->heap.destroy(g->drv); // no-op when the heap was never created
  g->ctrl.shutdown();
  delete g;
  g = nullptr;
}

// Test hook (B200MPI_EPOCH_START = e): give this rank's control region the state of a long-running job
// about to launch epoch e instead of zeros.  Every slot cell holds the oldest value a scrubbed row may
// hold, every slot flag e - 1, every ring step counter the value of one launch earlier.  The LL lanes
// stay zero, as a job's lanes beyond its largest message are.  Peers first write into this heap after
// Init's final barrier, so the preset needs no synchronisation.
static int preset_control_region(uint32_t e) {
  std::vector<Slot> slots((size_t)kMaxBlocks * kMaxRanks);
  const uint32_t oldest = e - kScrubEvery * kEpochStride;
  for (Slot& s : slots) {
    memset(&s, 0, sizeof s);
    for (uint4& cell : s.cell) cell = make_uint4(0, oldest, 0, oldest);
    s.flag = e - 1;
  }
  const std::vector<uint32_t> ring(kMaxBlocks, (e - kEpochStride) * 8u);
  char* base = (char*)g->heap.base[g->ctrl.rank];
  CUDA_OK(cudaMemcpy(base, slots.data(), slots.size() * sizeof(Slot), cudaMemcpyHostToDevice));
  CUDA_OK(cudaMemcpy(base + kRingFlagsOff, ring.data(), ring.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  CUDA_OK(cudaDeviceSynchronize());
  return 0;
}

int b200mpi_init(const char* addr, const char* alladdr_csv, const char* password, int64_t timeout_ns, int gpu) {
  std::lock_guard<std::mutex> lock(g_mu);
  if (g && g->initialised) return fail(B200MPI_ERR_ARG, "mpi: Init called twice");
  delete g;
  g = new Ctx();
  std::string err;
  int rc = g->ctrl.init(addr, alladdr_csv, password, timeout_ns, err);
  if (rc) { delete g; g = nullptr; return fail(rc, err); }
  if (const char* w = getenv("B200MPI_WATCHDOG_S")) g->watchdog_ns = (int64_t)(atof(w) * 1e9);
  // tell nobody: peers notice through their own control-plane errors / timeouts
  auto bail = [&](int code, const std::string& m) { teardown(); return fail(code, m); };
  if (gpu == -2) {
    g->control_only = true;
    settle_knobs();
    g->initialised = true;
    return 0;
  }
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0) {
    (void)cudaGetLastError();
    return bail(B200MPI_ERR_NO_DEVICE, std::string("no usable CUDA device: ") + (ce == cudaSuccess ? "device count is 0" : cudaGetErrorString(ce)) + " (libb200mpi has no CPU fallback)");
  }
  g->dev = gpu >= 0 ? gpu : g->ctrl.rank % ndev;
  if (g->dev >= ndev) return bail(B200MPI_ERR_ARG, "gpu ordinal " + std::to_string(g->dev) + " out of range (" + std::to_string(ndev) + " devices)");
  if ((ce = cudaSetDevice(g->dev)) != cudaSuccess || (ce = cudaFree(0)) != cudaSuccess)
    return bail(B200MPI_ERR_CUDA, std::string("cudaSetDevice: ") + cudaGetErrorString(ce));
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, g->dev);
  g->sm_count = prop.multiProcessorCount;
  if (prop.major != 9 || prop.minor != 0) return bail(B200MPI_ERR_NO_DEVICE, std::string("device '") + prop.name + "' is not sm_90 (H100-class); this library ships sm_90a code only");
  if (!g->drv.load(err)) return bail(B200MPI_ERR_CUDA, err);
  if (!(getenv("B200MPI_NUMA") && atoi(getenv("B200MPI_NUMA")) == 0)) g->gpu_numa_node = numa_node_of_gpu(g->dev);
  CounterEnv cenv;
  const std::string cenv_err = parse_counter_env(getenv("B200MPI_SCRUB_EVERY"), getenv("B200MPI_EPOCH_START"), getenv("B200MPI_LL_SEQ_START"),
                                                 kScrubEvery, kEpochStride, cenv);
  g->scrub_every = cenv.scrub_every;
  g->epoch = cenv.epoch_start;
  g->ll_seq = cenv.ll_seq_start;

  // who sits where: ranks sharing a device (functional-test mode) rule out NVLS.  The counter settings
  // travel along: ranks that disagree on them (or a rank that could not parse them) fail Init on every
  // rank instead of hanging in the first collective.
  struct Hello { unsigned char uuid[16]; int32_t dev; int32_t mc; uint32_t epoch_start, ll_seq_start, env_ok; } mine = {}, all[B200MPI_MAX_RANKS];
  memcpy(mine.uuid, &prop.uuid, 16);
  mine.dev = g->dev;
  int mc = 0;
  g->drv.DeviceGetAttribute(&mc, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, g->dev);
  mine.mc = mc;
  mine.epoch_start = cenv.epoch_start;
  mine.ll_seq_start = cenv.ll_seq_start;
  mine.env_ok = cenv_err.empty() ? 1u : 0u;
  rc = g->ctrl.allgather(&mine, sizeof mine, all, err);
  if (rc) return bail(rc, err);
  if (!cenv_err.empty()) return bail(B200MPI_ERR_ARG, cenv_err);
  for (int a = 0; a < g->ctrl.n; ++a) {
    if (!all[a].env_ok) return bail(B200MPI_ERR_ARG, "rank " + std::to_string(a) + " rejected its B200MPI_SCRUB_EVERY / B200MPI_EPOCH_START / B200MPI_LL_SEQ_START");
    if (all[a].epoch_start != mine.epoch_start || all[a].ll_seq_start != mine.ll_seq_start)
      return bail(B200MPI_ERR_ARG, "ranks disagree on B200MPI_EPOCH_START / B200MPI_LL_SEQ_START: rank " + std::to_string(a) + " has " +
                                       std::to_string(all[a].epoch_start) + " / " + std::to_string(all[a].ll_seq_start) + ", this rank " +
                                       std::to_string(mine.epoch_start) + " / " + std::to_string(mine.ll_seq_start));
  }
  bool want_nvls = g->ctrl.n > 1;
  if (const char* w = getenv("B200MPI_NVLS")) want_nvls = want_nvls && atoi(w) != 0;
  for (int a = 0; a < g->ctrl.n; ++a) {
    if (!all[a].mc) want_nvls = false;
    for (int b = a + 1; b < g->ctrl.n; ++b)
      if (memcmp(all[a].uuid, all[b].uuid, 16) == 0) g->shared_device = true;
  }
  if (g->shared_device) want_nvls = false;
  if (g->shared_device && !getenv("B200MPI_WATCHDOG_S")) g->watchdog_ns = 600ll * 1000000000ll; // time-sliced flags are slow

  size_t heap_bytes = 2ull << 30;
  if (const char* w = getenv("B200MPI_HEAP_BYTES")) heap_bytes = strtoull(w, nullptr, 0);
  if (heap_bytes < (64u << 20)) heap_bytes = 64u << 20;
  rc = g->heap.create(g->drv, g->ctrl, g->dev, heap_bytes, want_nvls, err);
  if (rc) return bail(rc, err);

  // mailbox shared memory
  {
    int mfd = -1, got = -1;
    if (g->ctrl.rank == 0) {
      mfd = memfd_create("b200mpi-mailbox", 0);
      if (mfd < 0 || ftruncate(mfd, sizeof(Mailbox)) != 0) return bail(B200MPI_ERR_BOOTSTRAP, std::string("mailbox memfd: ") + strerror(errno));
    }
    if (g->ctrl.n > 1) {
      rc = g->ctrl.bcast_fd(0, mfd, got, err);
      if (rc) return bail(rc, err);
    } else got = dup(mfd);
    void* m = mmap(nullptr, sizeof(Mailbox), PROT_READ | PROT_WRITE, MAP_SHARED, got, 0);
    if (mfd >= 0) close(mfd);
    close(got);
    if (m == MAP_FAILED) return bail(B200MPI_ERR_BOOTSTRAP, std::string("mailbox mmap: ") + strerror(errno));
    g->box = (Mailbox*)m; // zero-filled by ftruncate == every slot kFree
  }
  if (cudaHostAlloc((void**)&g->status_host, 64, cudaHostAllocMapped) != cudaSuccess ||
      cudaHostGetDevicePointer((void**)&g->status_dev, g->status_host, 0) != cudaSuccess)
    return bail(B200MPI_ERR_CUDA, "status word allocation failed");
  *g->status_host = 0;
  cudaStreamCreateWithFlags(&g->own_stream, cudaStreamNonBlocking);
  cudaStreamCreateWithFlags(&g->h2d_stream, cudaStreamNonBlocking);
  cudaStreamCreateWithFlags(&g->d2h_stream, cudaStreamNonBlocking);
  g->stream = g->own_stream;
  cudaEventCreate(&g->ev0);
  cudaEventCreate(&g->ev1);
  for (int r = 0; r < g->ctrl.n; ++r) g->comm.base[r] = (char*)g->heap.base[r];
  g->comm.mc = (char*)g->heap.mc_base;
  g->comm.status = g->status_dev;
  g->comm.timeout_ns = (unsigned long long)g->watchdog_ns;
  g->comm.rank = g->ctrl.rank;
  g->comm.n = g->ctrl.n;
  settle_knobs();
  if (cenv.preset && preset_control_region(cenv.epoch_start)) return bail(B200MPI_ERR_CUDA, t_err);
  rc = g->ctrl.barrier(err);
  if (rc) return bail(rc, err);
  g->initialised = true;
  return 0;
}

int b200mpi_finalize(void) {
  std::lock_guard<std::mutex> lock(g_mu);
  if (!g || !g->initialised) return fail(B200MPI_ERR_NOT_INIT, "mpi: Finalize without Init");
  std::string err;
  if (!g->control_only) {
    cudaSetDevice(g->dev);
    cudaDeviceSynchronize();
  }
  g->ctrl.barrier(err); // nobody unmaps while a peer may still read
  teardown();
  return 0;
}

int b200mpi_alloc(size_t bytes, void** dptr) {
  int rc = need_data_plane();
  if (rc) return rc;
  if (!dptr) return fail(B200MPI_ERR_ARG, "alloc: NULL result pointer");
  size_t off;
  if (g->heap.alloc(bytes, off)) return fail(B200MPI_ERR_NOMEM, "symmetric heap exhausted (" + std::to_string(g->heap.used()) + " of " + std::to_string(g->heap.size) + " bytes in use; raise B200MPI_HEAP_BYTES)");
  *dptr = (char*)g->heap.base[g->ctrl.rank] + off;
  return 0;
}

int b200mpi_free(void* dptr) {
  int rc = need_data_plane();
  if (rc) return rc;
  if (!dptr) return 0;
  size_t off = (char*)dptr - (char*)g->heap.base[g->ctrl.rank];
  if (g->heap.free_off(off)) return fail(B200MPI_ERR_ARG, "free: pointer was not returned by b200mpi_alloc");
  return 0;
}

int b200mpi_host_alloc(size_t bytes, void** hptr) {
  int rc = need_data_plane();
  if (rc) return rc;
  if (!hptr) return fail(B200MPI_ERR_ARG, "host_alloc: NULL result pointer");
  return numa_host_alloc(bytes, hptr);
}
int b200mpi_host_free(void* hptr) {
  int rc = need_data_plane();
  if (rc) return rc;
  CUDA_OK(cudaFreeHost(hptr));
  return 0;
}
int b200mpi_memcpy(void* dst, const void* src, size_t bytes, int kind) {
  int rc = need_data_plane();
  if (rc) return rc;
  cudaMemcpyKind k = kind == 0 ? cudaMemcpyHostToDevice : kind == 1 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  CUDA_OK(cudaMemcpyAsync(dst, src, bytes, k, g->stream));
  CUDA_OK(cudaStreamSynchronize(g->stream));
  return 0;
}
// Measured bound of the host-slice paths: plain pinned copies between a NUMA-local pinned buffer and
// the device heap, no collective.  bidir = H2D and D2H of `bytes` each running at the same time
// (what a pipelined host-slice Allreduce needs), reported per direction.
int b200mpi_pcie_probe(size_t bytes, int iters, double* h2d_gbs, double* d2h_gbs, double* bidir_gbs) {
  int rc = need_data_plane();
  if (rc) return rc;
  if (bytes == 0 || iters < 1) return fail(B200MPI_ERR_ARG, "pcie_probe: bytes and iters must be positive");
  void *ha = nullptr, *hb = nullptr;
  if ((rc = numa_host_alloc(bytes, &ha)) || (rc = numa_host_alloc(bytes, &hb))) { if (ha) cudaFreeHost(ha); return rc; }
  memset(ha, 1, bytes);
  size_t oa = 0, ob = 0;
  if (g->heap.alloc(bytes, oa) || g->heap.alloc(bytes, ob)) {
    cudaFreeHost(ha); cudaFreeHost(hb);
    return fail(B200MPI_ERR_NOMEM, "pcie_probe: symmetric heap exhausted");
  }
  char* da = (char*)g->heap.base[g->ctrl.rank] + oa;
  char* db = (char*)g->heap.base[g->ctrl.rank] + ob;
  auto timed = [&](bool up, bool down) {
    cudaStreamSynchronize(g->h2d_stream);
    cudaStreamSynchronize(g->d2h_stream);
    const auto t0 = Clock::now();
    for (int i = 0; i < iters; ++i) {
      if (up) cudaMemcpyAsync(da, ha, bytes, cudaMemcpyHostToDevice, g->h2d_stream);
      if (down) cudaMemcpyAsync(hb, db, bytes, cudaMemcpyDeviceToHost, g->d2h_stream);
    }
    cudaStreamSynchronize(g->h2d_stream);
    cudaStreamSynchronize(g->d2h_stream);
    const double sec = std::chrono::duration<double>(Clock::now() - t0).count();
    return (double)bytes * iters / sec / 1e9;
  };
  timed(true, true); // warm-up
  const double up = timed(true, false), down = timed(false, true), both = timed(true, true);
  if (h2d_gbs) *h2d_gbs = up;
  if (d2h_gbs) *d2h_gbs = down;
  if (bidir_gbs) *bidir_gbs = both;
  g->heap.free_off(oa);
  g->heap.free_off(ob);
  cudaFreeHost(ha);
  cudaFreeHost(hb);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(B200MPI_ERR_CUDA, std::string("pcie_probe: ") + cudaGetErrorString(e));
  return 0;
}
// Raw NVLink rates seen by this library's copy kernel between neighbouring ranks (the roofline the
// P2P collectives are held against).  Collective call.  mode 0: every rank pulls `bytes` from rank+1;
// 1: every rank pushes to rank+1; 2: only rank 0 pulls from rank 1; 3: only rank 0 pushes to rank 1;
// 4: every rank pulls from and pushes to rank+1 at the same time (two streams).
// *ms = device time of one iteration on this rank (0 for idle ranks).
int b200mpi_link_probe(size_t bytes, int mode, int iters, float* ms) {
  int rc = need_data_plane();
  if (rc) return rc;
  const int n = g->ctrl.n, me = g->ctrl.rank;
  if (n < 2 || bytes == 0 || iters < 1 || mode < 0 || mode > 4 || !ms) return fail(B200MPI_ERR_ARG, "link_probe: needs >= 2 ranks, bytes, iters >= 1, mode 0..4");
  size_t a = 0, b = 0;
  if (g->heap.alloc(bytes, a) || g->heap.alloc(bytes, b)) return fail(B200MPI_ERR_NOMEM, "link_probe: symmetric heap exhausted");
  struct Offs { uint64_t a, b; } mine = {a, b}, all[B200MPI_MAX_RANKS];
  std::string err;
  if ((rc = g->ctrl.allgather(&mine, sizeof mine, all, err))) return fail(rc, err);
  const int peer = (me + 1) % n;
  char* my_a = (char*)g->heap.base[me] + a;
  char* my_b = (char*)g->heap.base[me] + b;
  char* peer_a = (char*)g->heap.base[peer] + all[peer].a;
  char* peer_b = (char*)g->heap.base[peer] + all[peer].b;
  const bool active = mode == 0 || mode == 1 || mode == 4 || me == 0;
  cudaStream_t s2 = g->h2d_stream;
  CUDA_OK(cudaStreamSynchronize(g->stream));
  if ((rc = g->ctrl.barrier(err))) return fail(rc, err);
  *ms = 0.f;
  if (active) {
    for (int pass = 0; pass < 2; ++pass) { // pass 0 warms up
      const int k = pass ? iters : 2;
      CUDA_OK(cudaEventRecord(g->ev0, g->stream));
      if (mode == 4) CUDA_OK(cudaStreamWaitEvent(s2, g->ev0, 0));
      for (int i = 0; i < k && rc == 0; ++i) {
        if (mode == 0 || mode == 2 || mode == 4) rc = launch_copy(my_a, peer_a, bytes, g->stream);          // pull: loads cross the link
        if (rc == 0 && (mode == 1 || mode == 3)) rc = launch_copy(peer_b, my_b, bytes, g->stream);           // push: stores cross the link
        if (rc == 0 && mode == 4) rc = launch_copy(peer_b, my_b, bytes, s2);
      }
      if (rc) break;
      if (mode == 4) {
        cudaEvent_t e = g->pipe_events.empty() ? nullptr : g->pipe_events[0];
        if (!e) { CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); g->pipe_events.push_back(e); }
        CUDA_OK(cudaEventRecord(e, s2));
        CUDA_OK(cudaStreamWaitEvent(g->stream, e, 0));
      }
      CUDA_OK(cudaEventRecord(g->ev1, g->stream));
      CUDA_OK(cudaEventSynchronize(g->ev1));
      float t = 0;
      CUDA_OK(cudaEventElapsedTime(&t, g->ev0, g->ev1));
      *ms = t / k;
    }
  }
  std::string err2;
  g->ctrl.barrier(err2); // nobody frees while a neighbour still copies
  g->heap.free_off(a);
  g->heap.free_off(b);
  return rc;
}
int b200mpi_numa_node(void) { return (g && g->initialised && !g->control_only) ? g->gpu_numa_node : -1; }
int b200mpi_heap_info(size_t* total, size_t* used, int* nvls) {
  int rc = need_data_plane();
  if (rc) return rc;
  if (total) *total = g->heap.size;
  if (used) *used = g->heap.used();
  if (nvls) *nvls = g->heap.mc_base ? 1 : 0;
  return 0;
}

int b200mpi_send(const void* buf, size_t count, int dtype, int dest, int tag, int memkind) { return do_send(buf, count, dtype, dest, tag, memkind, true); }
int b200mpi_isend(const void* buf, size_t count, int dtype, int dest, int tag, int memkind) { return do_send(buf, count, dtype, dest, tag, memkind, false); }
int b200mpi_wait(int dest, int tag) { return do_wait(dest, tag); }
int b200mpi_recv(void* buf, size_t capacity, size_t* count_out, int dtype, int src, int tag, int memkind) { return do_recv(buf, capacity, count_out, dtype, src, tag, memkind); }

int b200mpi_bcast(void* buf, size_t count, int dtype, int root, int memkind) { return do_bcast(buf, count, dtype, root, memkind, false); }
int b200mpi_allreduce(const void* send, void* recv, size_t count, int dtype, int op, int memkind) { return do_allreduce(send, recv, count, dtype, op, memkind, false); }
int b200mpi_allgather(const void* send, void* recv, size_t count, int dtype, int memkind) { return do_allgather(send, recv, count, dtype, memkind, false); }
int b200mpi_reduce_scatter(const void* send, void* recv, size_t count_per_rank, int dtype, int op, int memkind) { return do_reduce_scatter(send, recv, count_per_rank, dtype, op, memkind, false); }
int b200mpi_reduce(const void* send, void* recv, size_t count, int dtype, int op, int root, int memkind) { return do_reduce(send, recv, count, dtype, op, root, memkind, false); }
int b200mpi_alltoall(const void* send, void* recv, size_t count_per_rank, int dtype, int memkind) { return do_alltoall(send, recv, count_per_rank, dtype, memkind, false); }
int b200mpi_scan(const void* send, void* recv, size_t count, int dtype, int op, int memkind) { return do_scan(send, recv, count, dtype, op, memkind, false); }
int b200mpi_exscan(const void* send, void* recv, size_t count, int dtype, int op, int memkind) { return do_scan(send, recv, count, dtype, op, memkind, true); }
int b200mpi_allreduce_loc(const void* send, void* recv, size_t count, int dtype, int op, int memkind) {
  return do_allreduce_loc(send, recv, count, dtype, op, 0, memkind, true);
}
int b200mpi_reduce_loc(const void* send, void* recv, size_t count, int dtype, int op, int root, int memkind) {
  return do_allreduce_loc(send, recv, count, dtype, op, root, memkind, false);
}
int b200mpi_win_create(void* base, size_t bytes, int* win) { return do_win_create(base, bytes, win); }
int b200mpi_win_free(int win) { return do_win_fence(win, true); }
int b200mpi_win_fence(int win) { return do_win_fence(win, false); }
int b200mpi_put(const void* origin, size_t count, int dtype, int target, size_t target_disp, int win, int memkind) {
  return do_rma(kPut, origin, count, dtype, 0, target, target_disp, win, memkind);
}
int b200mpi_get(void* origin, size_t count, int dtype, int target, size_t target_disp, int win, int memkind) {
  return do_rma(kGet, origin, count, dtype, 0, target, target_disp, win, memkind);
}
int b200mpi_accumulate(const void* origin, size_t count, int dtype, int op, int target, size_t target_disp, int win, int memkind) {
  return do_rma(kAccumulate, origin, count, dtype, op, target, target_disp, win, memkind);
}
int b200mpi_win_lock(int lock_type, int target, int win) { return do_win_lock(lock_type, target, win); }
int b200mpi_win_unlock(int target, int win) { return do_win_unlock(target, win); }
int b200mpi_get_accumulate(const void* origin, void* result, size_t count, int dtype, int op, int target, size_t target_disp, int win, int memkind) {
  return do_get_accumulate(origin, result, count, dtype, op, target, target_disp, win, memkind);
}
int b200mpi_fetch_and_op(const void* origin, void* result, int dtype, int op, int target, size_t target_disp, int win) {
  return do_fetch_and_op(origin, result, dtype, op, target, target_disp, win);
}
int b200mpi_compare_and_swap(const void* origin, const void* compare, void* result, int dtype, int target, size_t target_disp, int win) {
  return do_compare_and_swap(origin, compare, result, dtype, target, target_disp, win);
}
int b200mpi_win_post(const int* origins, int count, int win) { return do_win_post(origins, count, win); }
int b200mpi_win_start(const int* targets, int count, int win) { return do_win_start(targets, count, win); }
int b200mpi_win_complete(int win) { return do_win_complete(win); }
int b200mpi_win_wait(int win) { return do_win_wait(win, nullptr, false); }
int b200mpi_win_test(int win, int* flag) { return do_win_wait(win, flag, true); }
int b200mpi_gather(const void* send, void* recv, size_t count_per_rank, int dtype, int root, int memkind) { return do_gather(send, recv, count_per_rank, dtype, root, memkind, false); }
int b200mpi_scatter(const void* send, void* recv, size_t count_per_rank, int dtype, int root, int memkind) { return do_gather(send, recv, count_per_rank, dtype, root, memkind, true); }
int b200mpi_gatherv(const void* send, void* recv, const size_t* counts, int dtype, int root, int memkind) { return do_gatherv(send, recv, counts, dtype, root, false, memkind); }
int b200mpi_scatterv(const void* send, void* recv, const size_t* counts, int dtype, int root, int memkind) { return do_scatterv(send, recv, counts, dtype, root, memkind); }
int b200mpi_allgatherv(const void* send, void* recv, const size_t* counts, int dtype, int memkind) { return do_gatherv(send, recv, counts, dtype, 0, true, memkind); }
int b200mpi_reduce_scatterv(const void* send, void* recv, const size_t* counts, int dtype, int op, int memkind) {
  return do_reduce_scatterv(send, recv, counts, dtype, op, memkind);
}
int b200mpi_alltoallv(const void* send, const size_t* send_counts, void* recv, const size_t* recv_counts, int dtype, int memkind) {
  return do_alltoallv(send, send_counts, recv, recv_counts, dtype, memkind);
}
int b200mpi_reduce_scatter_async(const void* send, void* recv, size_t count_per_rank, int dtype, int op) { return do_reduce_scatter(send, recv, count_per_rank, dtype, op, B200MPI_DEVICE, true); }
int b200mpi_bcast_async(void* buf, size_t count, int dtype, int root) { return do_bcast(buf, count, dtype, root, B200MPI_DEVICE, true); }
int b200mpi_allreduce_async(const void* send, void* recv, size_t count, int dtype, int op) { return do_allreduce(send, recv, count, dtype, op, B200MPI_DEVICE, true); }
int b200mpi_allgather_async(const void* send, void* recv, size_t count, int dtype) { return do_allgather(send, recv, count, dtype, B200MPI_DEVICE, true); }

int b200mpi_stream_sync(void) {
  int rc = need_data_plane();
  if (rc) return rc;
  CUDA_OK(cudaStreamSynchronize(g->stream));
  return check_status();
}

int b200mpi_barrier(void) {
  if (int rc = need_init()) return rc;
  if (g->control_only) {
    std::string err;
    int rc = g->ctrl.barrier(err);
    return rc ? fail(rc, err) : 0;
  }
  if (g->ctrl.n == 1) return finish(false);
  int rc = launch_barrier(g->stream);
  if (rc) return rc;
  return finish(false);
}

int b200mpi_set_algo(int coll, int algo) {
  if (int rc = need_init()) return rc;
  if (coll < 0 || coll > B200MPI_COLL_REDUCE_SCATTER || algo < 0 || algo > B200MPI_ALGO_HYBRID) return fail(B200MPI_ERR_ARG, "set_algo: bad collective or algorithm id");
  g->algo[coll] = algo;
  return 0;
}
int b200mpi_get_algo(int coll, size_t count, int dtype) {
  int rc = need_data_plane();
  if (rc) return rc;
  const size_t bytes = count * esize(dtype);
  if (coll == B200MPI_COLL_ALLREDUCE) return pick_allreduce(bytes, dtype, B200MPI_SUM);
  if (coll == B200MPI_COLL_BCAST) return pick_bcast(bytes);
  if (coll == B200MPI_COLL_ALLGATHER) return pick_allgather(bytes);
  if (coll == B200MPI_COLL_REDUCE_SCATTER) return pick_reduce_scatter(bytes, dtype, B200MPI_SUM);
  return fail(B200MPI_ERR_ARG, "get_algo: bad collective id");
}
int b200mpi_set_param(const char* name, int64_t value) {
  if (int rc = need_init()) return rc;
  const Knob* k = find_knob(name);
  if (!k || k >= find_knob("sm_count")) return fail(B200MPI_ERR_ARG, std::string("set_param: unknown parameter '") + (name ? name : "") + "'");
  if (k->field == KnobField(&Ctx::host_threads) && g->pool.running())
    return fail(B200MPI_ERR_ARG, "set_param: host_threads must be set before the first pageable host-slice call");
  store_knob(*k, value);
  if (k->field == KnobField(&Ctx::watchdog_ns)) g->comm.timeout_ns = (unsigned long long)g->watchdog_ns;
  // leaving host_register mode drops every cached registration: the caller may free those buffers now
  if (k->field == KnobField(&Ctx::host_register) && !g->host_register) drop_registrations();
  return 0;
}
int b200mpi_get_param(const char* name, int64_t* value) {
  if (int rc = need_init()) return rc;
  if (!value) return fail(B200MPI_ERR_ARG, "get_param: NULL result pointer");
  const Knob* k = find_knob(name);
  if (!k) return fail(B200MPI_ERR_ARG, std::string("get_param: unknown parameter '") + (name ? name : "") + "'");
  *value = std::visit([&](auto m) { return (int64_t)(g->*m) / k->scale; }, k->field);
  return 0;
}
int b200mpi_set_max_blocks(int blocks) {
  if (int rc = need_init()) return rc;
  if (blocks < 0 || blocks > kMaxBlocks) return fail(B200MPI_ERR_ARG, "set_max_blocks: out of range");
  g->max_blocks = blocks; // block_cap() clamps to the SM count: the cross-rank barriers need every CTA resident
  return 0;
}
int b200mpi_get_stream(void** stream) {
  int rc = need_data_plane();
  if (rc) return rc;
  *stream = (void*)g->stream;
  return 0;
}
int b200mpi_set_stream(void* stream) {
  int rc = need_data_plane();
  if (rc) return rc;
  CUDA_OK(cudaStreamSynchronize(g->stream));
  g->stream = stream ? (cudaStream_t)stream : g->own_stream;
  return 0;
}
int b200mpi_timer_start(void) {
  int rc = need_data_plane();
  if (rc) return rc;
  CUDA_OK(cudaEventRecord(g->ev0, g->stream));
  return 0;
}
int b200mpi_timer_stop(float* ms) {
  int rc = need_data_plane();
  if (rc) return rc;
  CUDA_OK(cudaEventRecord(g->ev1, g->stream));
  CUDA_OK(cudaEventSynchronize(g->ev1));
  CUDA_OK(cudaEventElapsedTime(ms, g->ev0, g->ev1));
  return check_status();
}

} // extern "C"
