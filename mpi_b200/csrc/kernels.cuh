// kernels.cuh -- sm_90a (H100) device code of libb200mpi: the data plane that replaces the
// reference's gob-over-TCP Send/Receive (/root/reference/network.go:518-625) and implements the
// collectives the reference only stubs (/root/reference/mpi.go:130).
//
// Memory model.  Every rank owns one cuMem heap; all heaps are mapped into every rank's address
// space (Comm::base[r]) so a kernel reaches rank r's memory with plain ld/st.global that the
// GPU routes over NVLink 4 / NVSwitch (or stays local when r is this rank or shares the device).
// The first kCtrlBytes of each heap are control words:
//     Slot slots[kMaxBlocks][kMaxRanks]   cross-rank flag + per-call buffer descriptor
//     u32  ring[kMaxBlocks]               ring step counters
//     LL cells (kLLOff), window cells: lock word and PSCW counters (kWinLockOff)
// A collective kernel is   sync_start -> body -> sync_end   where both syncs are per-CTA
// barriers between the CTAs with the same blockIdx on every rank (flag writes with
// st.release.sys into the peer's slot, ld.acquire.sys spins on the own slot).  sync_start also
// carries this rank's {send,recv} heap offsets for the call, so user buffers may sit at
// different offsets on different ranks.  Epochs only grow; comparisons are wrap-safe.
//
// Reduction order (what oracle/collectives.c restates, bit for bit):
//   one-shot / two-shot : acc = x_0; acc = op(acc, x_r) for r = 1..n-1          ("rank order")
//   one-shot shuffle    : pairwise tree ((x0+x1)+(x2+x3))+((x4+x5)+(x6+x7))      ("tree order")
//   ring                : chunk c: ((x_c + x_{c+1}) + ...) + x_{c-1}  (cyclic from c) ("ring order")
//   nvls                : order chosen by the switch (tolerance-checked for floats, exact for ints)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <type_traits>

namespace b200 {

constexpr int kMaxRanks = 8;
constexpr int kMaxBlocks = 528;            // 132 SMs x 4
constexpr size_t kCtrlBytes = 16u << 20;   // control region at the start of every heap (== kHeapReserved, heap.h)
constexpr size_t kRingFlagsOff = 512u << 10;
constexpr size_t kLLStateOff = 768u << 10;   // LL bookkeeping words (device-resident sequence number, CTA counter)
constexpr size_t kLLOff = 1u << 20;          // LL cells: [parity 2][src rank n][ll_cells(n)] x 16 B, 8 MiB in all
constexpr size_t kLLRegionCells = 2 * 8 * 32768;
// cells per lane: 8 payload bytes each -> 256 KiB per call at n = 8, 512 KiB at n = 4, 1 MiB at n = 2
__host__ __device__ constexpr size_t ll_cells(int n) { return kLLRegionCells / (2 * (size_t)(n < 1 ? 1 : n)); }
constexpr int kThreads = 512;
// Every collective launch consumes exactly kEpochStride flag values, whatever the algorithm:
// start barrier = epoch, mid barriers = epoch+1 .. epoch+kEpochStride-2, end barrier =
// epoch+kEpochStride-1.  Ranks that disagreed about a call (B200MPI_ERR_PEER) therefore still
// agree about the epoch of the next one.
constexpr uint32_t kEpochStride = 4096;
constexpr uint32_t kMaxMids = kEpochStride - 2;
constexpr uint32_t kScrubEvery = 1u << 14;  // launches between two scrub_kernel runs (see there): barrier flags then lag by at most
                                            // 2^14 * 4096 = 2^26, ring step counters (epoch * 8) by 2^29, both far below 2^31

// One slot per (CTA, source rank).  The start barrier needs no release fence: the three cells are
// plain 16-byte stores that carry their own flag next to every 8 payload bytes (the LL idea: only
// 8-byte store atomicity is assumed), so a peer's {send offset, recv offset, signature} are valid
// as soon as all six flag words equal this call's epoch -- one NVLink one-way latency instead of a
// round trip (release = wait for the acks of the payload stores) plus a one-way.  `flag` is the
// release/acquire word of the mid and end barriers, where the body's stores must have landed.
struct __align__(64) Slot {
  uint4 cell[3];    // {lo32, epoch, hi32, epoch} of: a = writer's send offset, b = recv offset, c = signature
  uint32_t flag;
  uint32_t pad[3];
};
static_assert(sizeof(Slot) == 64, "slot size");
struct Comm {
  char* base[kMaxRanks];     // heap of rank r as mapped in this process
  char* mc;                  // multicast (NVLS) mapping of all heaps, or nullptr
  uint32_t* status;          // host-mapped word: != 0 after a device-side watchdog timeout
  unsigned long long timeout_ns;
  int rank, n;
  uint32_t epoch;            // start barrier value
  uint32_t end_epoch;        // end barrier value (epoch + 1 + number of reserved mid barriers)
  uint64_t sig;              // what this rank thinks the call is: (count, collective, dtype, op, algorithm)
};

// The splitmix64 finaliser, a bijection of 64-bit words: folds call signatures (b200mpi.cu:
// make_sig) and the Alltoallv table digest (a2av_tables).
__host__ __device__ inline uint64_t mix64(uint64_t x) {
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27; x *= 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

// The wrap-safe comparison of every barrier: flag word `v` has reached `want` when it is at most
// 2^31 - 1 ahead of it.  Sound only while no word lags the value it is compared with by 2^31 or
// more (scrub_kernel keeps it so).
__host__ __device__ __forceinline__ bool flag_reached(uint32_t v, uint32_t want) { return (int32_t)(v - want) >= 0; }
// flag_reached for six words at once.  A difference v - want has its sign bit set exactly when
// flag_reached(v, want) is false, so all six have reached `want` when the OR of their differences
// has a clear sign bit: six subtractions, three ORs and one sign test per poll, as the start
// barrier's spin compiled to when it was written out by hand.  (A chain of six flag_reached calls,
// with & or &&, compiles to longer code.)
__host__ __device__ __forceinline__ bool flags_reached(uint32_t v0, uint32_t v1, uint32_t v2, uint32_t v3, uint32_t v4, uint32_t v5, uint32_t want) {
  return flag_reached(want + ((v0 - want) | (v1 - want) | (v2 - want) | (v3 - want) | (v4 - want) | (v5 - want)), want);
}

// LL sequence numbers (allreduce_ll_kernel).  A peer's cell counts as arrived when both its flag
// words equal the call's sequence number, so a value must never meet a cell written 2^32 values
// earlier, nor the zeros of a cleared lane.  The next value after `last` when `step` are consumed
// (1 for an LL call, 2 for resync_after_error, which skips one value of each parity): never 0, and
// `wrapped` is set when the advance crosses 2^32.  The sequence then restarts at 1, and the caller
// must clear the LL lanes of every rank before the next LL kernel runs.
struct LLSeqNext { uint32_t seq; bool wrapped; };
__host__ __device__ inline LLSeqNext ll_seq_next(uint32_t last, uint32_t step) {
  const uint32_t v = last + step;
  if (v < last) return {1u, true}; // also covers landing on 0 exactly

  return {v, false};
}

// ---------------------------------------------------------------------------------------------
// flag primitives
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys_u64(uint64_t* p, uint64_t v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_relaxed_sys_u64(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// 16-byte cells that carry their own flag words (start barrier slots, LL lanes)
__device__ __forceinline__ void st_cell16(uint4* p, uint4 v) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 ld_cell16(const uint4* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}

// Spin until *p >= want (wrap-safe).  On watchdog expiry raises the host-visible status word
// and gives up so the kernel can drain; the host then reports B200MPI_ERR_TIMEOUT.  The poll is
// written out here, in wait_cells and in allreduce_ll_kernel: shared through one helper it
// compiled to different SASS in alltoallv_push_kernel and allreduce_ll_kernel.
__device__ __forceinline__ bool wait_flag(const uint32_t* p, uint32_t want, const Comm& c) {
  unsigned long long t0 = 0;
  uint32_t it = 0;
  while (!flag_reached(ld_acquire_sys(p), want)) {
    if ((++it & 0xfffu) == 0) {
      unsigned long long now = globaltimer_ns();
      if (t0 == 0) t0 = now;
      else if (c.timeout_ns && now - t0 > c.timeout_ns) {
        *(volatile uint32_t*)c.status = 1u;
        __threadfence_system();
        return false;
      }
    }
  }
  return true;
}

__device__ __forceinline__ Slot* slot_of(const Comm& c, int owner, int block, int src) {
  return reinterpret_cast<Slot*>(c.base[owner]) + (size_t)block * kMaxRanks + src;
}

// Spin until the three cells of `s` carry `epoch`; values out through a/b/sig.  false on watchdog expiry.
__device__ __forceinline__ bool wait_cells(const Slot* s, uint32_t epoch, const Comm& c, uint64_t& a, uint64_t& b, uint64_t& sig) {
  unsigned long long t0 = 0;
  uint32_t it = 0;
  for (;;) {
    const uint4 x = ld_cell16(&s->cell[0]), y = ld_cell16(&s->cell[1]), z = ld_cell16(&s->cell[2]);
    // >= (wrap-safe), not ==: in normal operation a peer is never ahead (it waits for this CTA at its end
    // barrier), so the two are the same; after a failed call a peer may already be announcing its next
    // one, and a late CTA must then see "newer, different signature" at once instead of spinning.
    if (flags_reached(x.y, x.w, y.y, y.w, z.y, z.w, epoch)) {
      a = ((uint64_t)x.z << 32) | x.x;
      b = ((uint64_t)y.z << 32) | y.x;
      sig = ((uint64_t)z.z << 32) | z.x;
      return true;
    }
    if ((++it & 0xfffu) == 0) {
      const unsigned long long now = globaltimer_ns();
      if (t0 == 0) t0 = now;
      else if (c.timeout_ns && now - t0 > c.timeout_ns) {
        *(volatile uint32_t*)c.status = 1u;
        __threadfence_system();
        return false;
      }
    }
  }
}

// Why sync_start said no, for sync_end_failed: 0 fine, 1 this CTA's partner announced a different
// signature (the partner exists and fails the same way), 2 a peer's CTA 0 announced a different
// signature (grids may differ: this CTA may have no partner at all), 3 watchdog.
__device__ __forceinline__ int* start_verdict() {
  __shared__ int verdict;
  return &verdict;
}

// The last step of both start barriers, once every thread sees the final verdict: true when the
// body may run; otherwise thread 0 raises status 2 (B200MPI_ERR_PEER) unless the watchdog has
// already raised status 1.
__device__ __forceinline__ bool start_agreed(const Comm& c) {
  const int v = *start_verdict();
  if (v) {
    if (threadIdx.x == 0 && v != 3) {
      *(volatile uint32_t*)c.status = 2u;
      __threadfence_system();
    }
    return false;
  }
  return true;
}

// Per-CTA barrier #1: announce {a,b,sig} to every rank, wait for everyone's, publish the offsets
// in smem.  Returns false when the body must not run:
//   * a peer's signature differs from ours (status 2 -> B200MPI_ERR_PEER): ranks called different
//     collectives / counts / types / grids, or
//   * a peer did not show up within the watchdog time (status 1 -> B200MPI_ERR_TIMEOUT).
// sync_end still runs, so nobody hangs, and no buffer is touched.
// The signature covers the grid size.  CTAs other than 0 first look at what every peer's CTA 0
// announced (slot row 0 of this rank's heap): if the peers launched a different grid, a CTA
// without a partner learns it there instead of waiting for a flag that never comes.  (While the
// grids match the row cannot be overwritten early: a peer's next kernel starts only after its
// current one has finished, which needs this CTA to have passed sync_end.)
__device__ __forceinline__ bool sync_start(const Comm& c, uint64_t a, uint64_t b, uint64_t* s_a,
                                           uint64_t* s_b) {
  int* verdict = start_verdict();
  const int t = threadIdx.x;
  if (t == 0) *verdict = 0;
  __syncthreads();
  if (t < c.n) {
    Slot* theirs = slot_of(c, t, blockIdx.x, c.rank);
    st_cell16(&theirs->cell[0], make_uint4((uint32_t)a, c.epoch, (uint32_t)(a >> 32), c.epoch));
    st_cell16(&theirs->cell[1], make_uint4((uint32_t)b, c.epoch, (uint32_t)(b >> 32), c.epoch));
    st_cell16(&theirs->cell[2], make_uint4((uint32_t)c.sig, c.epoch, (uint32_t)(c.sig >> 32), c.epoch));
    bool ok = true;
    uint64_t pa, pb, psig;
    if (blockIdx.x != 0) {
      if (!wait_cells(slot_of(c, c.rank, 0, t), c.epoch, c, pa, pb, psig)) { atomicMax(verdict, 3); ok = false; }
      else if (psig != c.sig) { atomicMax(verdict, 2); ok = false; }
    }
    if (ok) {
      if (!wait_cells(slot_of(c, c.rank, blockIdx.x, t), c.epoch, c, pa, pb, psig)) atomicMax(verdict, 3);
      else {
        s_a[t] = pa;
        s_b[t] = pb;
        if (psig != c.sig) atomicMax(verdict, 1);
      }
    }
  }
  __syncthreads();
  return start_agreed(c);
}

// The start barrier of a call whose ranks hold different tables (Alltoallv).  Thread t announces
// values meant for rank t alone: a_t = the bytes this rank expects from t, b_t = the heap offset where
// t's block lands here.  On return s_a[t] = the bytes t expects from this rank, s_b[t] = where this
// rank's block lands in t's heap.  The signatures differ from rank to rank (c.sig = base_sig + this
// rank's table digest): the call is well formed when the n announced words sum to n * base_sig.
// Every rank sums the same n words (each rank writes one signature into every slot row), so every
// rank reaches the same verdict -- over row 0 first for CTAs other than 0, as sync_start does, then
// over its own row.  Each pair also compares its byte counts exactly (s_a[t] against want_t), so even
// a digest collision could not let this rank write more than a peer expects.  Verdicts and exits are
// sync_start's, and sync_end / sync_end_failed follow as usual.
__device__ __forceinline__ bool sync_start_pairs(const Comm& c, uint64_t base_sig, uint64_t a_t, uint64_t b_t, uint64_t want_t,
                                                 uint64_t* s_a, uint64_t* s_b) {
  __shared__ unsigned long long sums[2]; // of row 0, of this CTA's row (mod 2^64)
  int* verdict = start_verdict();
  const int t = threadIdx.x;
  const unsigned long long want_sum = (unsigned long long)c.n * base_sig;
  if (t == 0) { *verdict = 0; sums[0] = 0; sums[1] = 0; }
  __syncthreads();
  uint64_t pa, pb, psig;
  if (t < c.n) {
    Slot* theirs = slot_of(c, t, blockIdx.x, c.rank);
    st_cell16(&theirs->cell[0], make_uint4((uint32_t)a_t, c.epoch, (uint32_t)(a_t >> 32), c.epoch));
    st_cell16(&theirs->cell[1], make_uint4((uint32_t)b_t, c.epoch, (uint32_t)(b_t >> 32), c.epoch));
    st_cell16(&theirs->cell[2], make_uint4((uint32_t)c.sig, c.epoch, (uint32_t)(c.sig >> 32), c.epoch));
    if (blockIdx.x != 0) {
      if (!wait_cells(slot_of(c, c.rank, 0, t), c.epoch, c, pa, pb, psig)) atomicMax(verdict, 3);
      else atomicAdd(&sums[0], (unsigned long long)psig);
    }
  }
  __syncthreads();
  if (t == 0 && blockIdx.x != 0 && *verdict == 0 && sums[0] != want_sum) *verdict = 2;
  __syncthreads();
  if (t < c.n && *verdict == 0) {
    if (!wait_cells(slot_of(c, c.rank, blockIdx.x, t), c.epoch, c, pa, pb, psig)) atomicMax(verdict, 3);
    else {
      s_a[t] = pa;
      s_b[t] = pb;
      atomicAdd(&sums[1], (unsigned long long)psig);
      if (pa != want_t) atomicMax(verdict, 1);
    }
  }
  __syncthreads();
  if (t == 0 && *verdict == 0 && sums[1] != want_sum) *verdict = 1;
  __syncthreads();
  return start_agreed(c);
}

// Per-CTA barrier #2: all of this CTA's stores (local, peer and multicast) are released to every
// rank, and every rank's matching CTA has finished reading/writing this rank's buffers.
__device__ __forceinline__ void sync_end(const Comm& c) {
  __syncthreads();
  const int t = threadIdx.x;
  if (t < c.n) {
    st_release_sys(&slot_of(c, t, blockIdx.x, c.rank)->flag, c.end_epoch);
    wait_flag(&slot_of(c, c.rank, blockIdx.x, t)->flag, c.end_epoch, c);
  }
}

// The way out of a kernel whose sync_start said no (the body was skipped, nothing of this CTA is in
// flight).  The end flag is always signalled, so a partner that is waiting gets released; this CTA
// itself waits only when it knows a partner exists and left the same way (verdict 1) -- a CTA that
// learnt about the mismatch from the peers' CTA 0, or that timed out, may have no partner, and
// waiting for one would stall until the watchdog.
__device__ __forceinline__ void sync_end_failed(const Comm& c) {
  __syncthreads();
  const int t = threadIdx.x;
  const bool wait = *start_verdict() == 1;
  if (t < c.n) {
    st_release_sys(&slot_of(c, t, blockIdx.x, c.rank)->flag, c.end_epoch);
    if (wait) wait_flag(&slot_of(c, c.rank, blockIdx.x, t)->flag, c.end_epoch, c);
  }
}

// Per-CTA barrier between a read phase and a write phase of the same addresses (in-place
// one-shot): `value` must lie strictly between c.epoch and c.end_epoch and grow from call to call.
__device__ __forceinline__ void sync_mid(const Comm& c, uint32_t value) {
  __syncthreads();
  const int t = threadIdx.x;
  if (t < c.n) {
    st_release_sys(&slot_of(c, t, blockIdx.x, c.rank)->flag, value);
    wait_flag(&slot_of(c, c.rank, blockIdx.x, t)->flag, value, c);
  }
  __syncthreads();
}

// The frame of a collective kernel: sync_start announcing this rank's offsets a and b, then
// body(s_a, s_b) with every rank's offsets, then sync_end.  A refused call skips the body and leaves
// through sync_end_failed.  A CTA that left any other way would keep its peers waiting until the
// watchdog fires, so every kernel of that shape goes through here.
template <typename Body>
__device__ __forceinline__ void collective(const Comm& c, uint64_t a, uint64_t b, Body body) {
  __shared__ uint64_t s_a[kMaxRanks], s_b[kMaxRanks];
  if (!sync_start(c, a, b, s_a, s_b)) { // ranks disagree about this call: touch nothing, leave through the end barrier
    sync_end_failed(c);
    return;
  }
  body(s_a, s_b);
  sync_end(c);
}

// ---------------------------------------------------------------------------------------------
// 16-byte packs
// ---------------------------------------------------------------------------------------------
template <typename T>
struct alignas(16) Pack {
  static constexpr int N = 16 / sizeof(T);
  T v[N];
};

__device__ __forceinline__ uint4 ldg16(const void* p) { // streaming 128-bit load (local or peer)
  uint4 r;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ void stg16(void* p, uint4 v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}
template <typename T>
__device__ __forceinline__ Pack<T> ld_pack(const void* p) {
  union { uint4 u; Pack<T> k; } x;
  x.u = ldg16(p);
  return x.k;
}
__device__ __forceinline__ uint4 ldg16_sys(const void* p) { // coherent at system scope: never served from L1
  uint4 r;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
template <typename T>
__device__ __forceinline__ Pack<T> ld_pack_sys(const void* p) {
  union { uint4 u; Pack<T> k; } x;
  x.u = ldg16_sys(p);
  return x.k;
}
template <typename T>
__device__ __forceinline__ void st_pack(void* p, const Pack<T>& v) {
  union { uint4 u; Pack<T> k; } x;
  x.k = v;
  stg16(p, x.u);
}

struct OpSum {
  template <typename T> __device__ __forceinline__ static T apply(T a, T b) { return a + b; }
};
template <> __device__ __forceinline__ long long OpSum::apply<long long>(long long a, long long b) {
  return (long long)((unsigned long long)a + (unsigned long long)b); // Go int64 wrap-around
}
struct OpMax {
  template <typename T> __device__ __forceinline__ static T apply(T a, T b) { return b > a ? b : a; }
};
struct OpMin {
  template <typename T> __device__ __forceinline__ static T apply(T a, T b) { return b < a ? b : a; }
};
// One-sided only (B200MPI_REPLACE, B200MPI_NO_OP): tags for Red and Fetch, never reduced with apply.
struct OpReplace {};
struct OpNoOp {};

// A value-location pair of MAXLOC / MINLOC: the C struct { V val; int64_t loc; }, 16 bytes for f32,
// f64 and i64 alike (4 padding bytes follow an f32 value).  `w` holds the value's bytes and the
// padding, so that a pair is always moved whole: the winner's value bits, loc and padding.
template <typename V>
struct Loc {
  unsigned long long w;
  long long loc;
  __host__ __device__ __forceinline__ V val() const {
    V v;
    memcpy(&v, &w, sizeof(V));
    return v;
  }
};
static_assert(sizeof(Loc<float>) == 16 && sizeof(Loc<double>) == 16 && sizeof(Loc<long long>) == 16, "pair size");

// MAXLOC (MAX) / MINLOC (!MAX) of a (the lower ranks) and b (a higher rank): b wins when its value is
// better, or equal with a smaller loc; on a tie of both a is kept.  Floats compare as IEEE (-0 == +0),
// except that a NaN is better than every number under both ops and equal to every other NaN.  The
// winner is the lowest-ranked pair among the best ones, so any bracketing of the fold agrees.
template <bool MAX, typename V>
__host__ __device__ __forceinline__ Loc<V> apply_loc(const Loc<V>& a, const Loc<V>& b) {
  const V x = a.val(), y = b.val();
  const bool xnan = x != x, ynan = y != y;
  const bool better = xnan ? false : ynan ? true : MAX ? y > x : y < x;
  const bool equal = xnan ? ynan : !ynan && x == y;
  return (better || (equal && b.loc < a.loc)) ? b : a;
}
struct OpMaxLoc {
  template <typename T> __host__ __device__ __forceinline__ static T apply(T a, T b) { return apply_loc<true>(a, b); }
};
struct OpMinLoc {
  template <typename T> __host__ __device__ __forceinline__ static T apply(T a, T b) { return apply_loc<false>(a, b); }
};

template <typename T, typename Op>
__device__ __forceinline__ Pack<T> combine(const Pack<T>& a, const Pack<T>& b) {
  Pack<T> r;
#pragma unroll
  for (int i = 0; i < Pack<T>::N; ++i) r.v[i] = Op::template apply<T>(a.v[i], b.v[i]);
  return r;
}

__device__ __forceinline__ bool all_aligned16(const uint64_t* s_a, const uint64_t* s_b, int n) {
  uint64_t m = 0;
  for (int r = 0; r < n; ++r) m |= s_a[r] | s_b[r];
  return (m & 15) == 0;
}

// Element e of the buffer at byte address p, loaded and stored through volatile accesses of the
// element's own width.  A pair has no volatile copy: it moves as two 8-byte halves.
template <typename T>
struct Elem {
  template <typename P> __device__ __forceinline__ static T ld(P p, size_t e) { return reinterpret_cast<const volatile T*>(p)[e]; }
  template <typename P> __device__ __forceinline__ static void st(P p, size_t e, T v) { reinterpret_cast<volatile T*>(p)[e] = v; }
};
template <typename V>
struct Elem<Loc<V>> {
  template <typename P> __device__ __forceinline__ static Loc<V> ld(P p, size_t e) {
    const volatile unsigned long long* q = reinterpret_cast<const volatile unsigned long long*>(p) + 2 * e;
    Loc<V> x;
    x.w = q[0];
    x.loc = (long long)q[1];
    return x;
  }
  template <typename P> __device__ __forceinline__ static void st(P p, size_t e, Loc<V> v) {
    volatile unsigned long long* q = reinterpret_cast<volatile unsigned long long*>(p) + 2 * e;
    q[0] = v.w;
    q[1] = (unsigned long long)v.loc;
  }
};

// Element e of the n buffers at byte addresses src(0), ..., src(n-1), reduced in rank order:
// acc = x_0; acc = op(acc, x_r) for r = 1..n-1.
template <typename T, typename Op, typename Src>
__device__ __forceinline__ T reduce_ranks(Src src, int n, size_t e) {
  T acc = Elem<T>::ld(src(0), e);
  for (int r = 1; r < n; ++r) acc = Op::template apply<T>(acc, Elem<T>::ld(src(r), e));
  return acc;
}
// ... of the n sends of a call (rank r's at heap offset s_a[r])
template <typename T, typename Op>
__device__ __forceinline__ T reduce_ranks(const Comm& c, const uint64_t* s_a, int n, size_t e) {
  return reduce_ranks<T, Op>([&](int r) { return c.base[r] + s_a[r]; }, n, e);
}

// Elements [lo, hi), CTA bid of nb working on them: each reduced over the n sends in rank order and
// stored, one element at a time, into every rank's recv (only_dst < 0) or into rank only_dst's.
template <typename T, typename Op>
__device__ __forceinline__ void reduce_store_elements(const Comm& c, const uint64_t* s_a, const uint64_t* s_b, int n, size_t lo, size_t hi,
                                                      unsigned bid, unsigned nb, int only_dst = -1) {
  const size_t gtid = (size_t)bid * blockDim.x + threadIdx.x;
  for (size_t e = lo + gtid; e < hi; e += (size_t)nb * blockDim.x) {
    const T acc = reduce_ranks<T, Op>(c, s_a, n, e);
    for (int r = 0; r < n; ++r)
      if (only_dst < 0 || r == only_dst) Elem<T>::st(c.base[r] + s_b[r], e, acc);
  }
}

// Rank `rank`'s contiguous share [lo, hi) of `count` elements cut into n equal parts (the last ones
// may be short or empty): element ownership of unaligned buffers.
struct Range {
  size_t lo, hi;
};
__device__ __forceinline__ Range owned_elements(size_t count, int n, int rank) {
  const size_t per = (count + n - 1) / n;
  const size_t lo = per * rank < count ? per * rank : count;
  return {lo, lo + per < count ? lo + per : count};
}

// The grid-strided copy loop of units [lo, hi): each thread loads UNROLL units (load(i, v)) before it
// stores any of them (store(i, v)), so UNROLL loads are in flight per thread.
template <int UNROLL, typename V, typename Load, typename Store>
__device__ __forceinline__ void unrolled(size_t lo, size_t hi, Load load, Store store) {
  const size_t step = (size_t)gridDim.x * blockDim.x * UNROLL;
  for (size_t i0 = lo + (size_t)blockIdx.x * blockDim.x * UNROLL + threadIdx.x; i0 < hi; i0 += step) {
    V v[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t i = i0 + (size_t)u * blockDim.x;
      if (i < hi) load(i, v[u]);
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t i = i0 + (size_t)u * blockDim.x;
      if (i < hi) store(i, v[u]);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Allreduce, one-shot: every rank reads all n buffers and keeps the whole result (latency path).
// The work is cut into rounds of one unit per thread.  When any rank runs in place
// (send == recv) a round is  read+reduce -> sync_mid -> write : nobody overwrites a value that a
// peer has yet to read.  Out of place the mid barriers are skipped.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool any_inplace(const uint64_t* s_a, const uint64_t* s_b, int n) {
  bool ip = false;
  for (int r = 0; r < n; ++r) ip = ip || s_a[r] == s_b[r];
  return ip;
}

template <typename T, typename Op, int NR>
__global__ void __launch_bounds__(kThreads, 1)
allreduce_oneshot_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t count) {
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    const int n = NR ? NR : c.n;
    const size_t gtid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t gstride = (size_t)gridDim.x * blockDim.x;
    char* out = c.base[c.rank] + s_b[c.rank];
    const bool inplace = any_inplace(s_a, s_b, n);
    uint32_t mid = c.epoch + 1;
    constexpr int EPV = Pack<T>::N;
    const bool al = all_aligned16(s_a, s_b, n);
    const size_t nvec = al ? count / EPV : 0;
    for (size_t base = 0; base < nvec; base += gstride) {
      const size_t i = base + gtid;
      Pack<T> acc;
      if (i < nvec) {
        Pack<T> v[NR ? NR : kMaxRanks];
#pragma unroll
        for (int r = 0; r < (NR ? NR : kMaxRanks); ++r)
          if (r < n) v[r] = ld_pack<T>(c.base[r] + s_a[r] + i * 16);
        acc = v[0];
#pragma unroll
        for (int r = 1; r < (NR ? NR : kMaxRanks); ++r)
          if (r < n) acc = combine<T, Op>(acc, v[r]);
      }
      if (inplace) sync_mid(c, mid++);
      if (i < nvec) st_pack<T>(out + i * 16, acc);
    }
    // scalar rounds: the count % EPV tail, or everything when some buffer is not 16-byte aligned
    for (size_t base = nvec * EPV; base < count; base += gstride) {
      const size_t e = base + gtid;
      T acc = T(0);
      if (e < count) acc = reduce_ranks<T, Op>(c, s_a, n, e);
      if (inplace) sync_mid(c, mid++);
      if (e < count) reinterpret_cast<T*>(out)[e] = acc;
    }
  });
}

// One-shot with a lane per peer and warp-shuffle partial sums (n = 2, 4, 8; tree order).
// 32/NR vectors per warp step; all NR peer loads of one vector are issued by different lanes in
// the same instruction, so a small message costs one NVLink round trip.
template <typename T, typename Op, int NR>
__global__ void __launch_bounds__(kThreads, 1)
allreduce_oneshot_shfl_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t count) {
  __shared__ const char* s_src[kMaxRanks];
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    if (threadIdx.x < NR) s_src[threadIdx.x] = c.base[threadIdx.x] + s_a[threadIdx.x];
    __syncthreads();
    constexpr int EPV = Pack<T>::N;
    constexpr int VPW = 32 / NR; // vectors per warp step
    const int lane = threadIdx.x & 31;
    const int peer = lane % NR, sub = lane / NR;
    const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
    char* out = c.base[c.rank] + s_b[c.rank];
    const bool al = all_aligned16(s_a, s_b, NR);
    const bool inplace = any_inplace(s_a, s_b, NR);
    uint32_t mid = c.epoch + 1;
    const size_t nvec = al ? count / EPV : 0;
    const char* src = s_src[peer];
    for (size_t round = 0; round < nvec; round += nwarps * VPW) { // uniform across the CTA
      const size_t i = round + warp * VPW + sub;
      const bool valid = i < nvec;
      Pack<T> v;
      if (valid) v = ld_pack<T>(src + i * 16);
      else
        for (int k = 0; k < EPV; ++k) v.v[k] = T(0);
#pragma unroll
      for (int m = 1; m < NR; m <<= 1) {
        union { Pack<T> k; uint32_t w[4]; } a, b;
        a.k = v;
#pragma unroll
        for (int w = 0; w < 4; ++w) b.w[w] = __shfl_xor_sync(0xffffffffu, a.w[w], m);
        v = (peer & m) ? combine<T, Op>(b.k, v) : combine<T, Op>(v, b.k); // lower ranks on the left
      }
      if (inplace) sync_mid(c, mid++);
      if (peer == 0 && valid) st_pack<T>(out + i * 16, v);
    }
    // scalar rounds (tail, or the whole message when unaligned), tree order too
    const size_t gtid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t gstride = (size_t)gridDim.x * blockDim.x;
    for (size_t base = nvec * EPV; base < count; base += gstride) {
      const size_t e = base + gtid;
      T x[NR];
      if (e < count) {
#pragma unroll
        for (int r = 0; r < NR; ++r) x[r] = reinterpret_cast<const volatile T*>(s_src[r])[e];
#pragma unroll
        for (int m = 1; m < NR; m <<= 1)
#pragma unroll
          for (int r = 0; r < NR; r += 2 * m) x[r] = Op::template apply<T>(x[r], x[r + m]);
      }
      if (inplace) sync_mid(c, mid++);
      if (e < count) reinterpret_cast<T*>(out)[e] = x[0];
    }
  });
}

// ---------------------------------------------------------------------------------------------
// Ownership of the message for the owner-reduces kernels (two-shot, smem two-shot, NVLS).
// The message is cut into blocks of 2^shift 16-byte vectors; block k belongs to rank k % n, so at
// any moment all n ranks work inside the same few-MiB window of every heap (fine interleave keeps
// DRAM pages, GPU TLBs and the switch's multicast tables hot; with one contiguous slice per rank
// NVLS lost 30% beyond 256 MiB).  The host picks `shift` from (count, n) only, so every rank
// agrees.  Results do not depend on it: each element is reduced exactly once, in rank order.
// ---------------------------------------------------------------------------------------------
struct Owner {
  size_t nvec;   // whole 16-byte vectors in the message
  size_t slots;  // upper bound of this rank's local vector slots: (blocks owned) << shift
  uint32_t shift;
  int n, rank;
  __host__ __device__ __forceinline__ Owner(size_t nvec_, uint32_t shift_, int n_, int rank_) : nvec(nvec_), shift(shift_), n(n_), rank(rank_) {
    const size_t nblk = (nvec_ + ((size_t)1 << shift_) - 1) >> shift_;
    const size_t mine = nblk > (size_t)rank_ ? (nblk - rank_ + n_ - 1) / n_ : 0;
    slots = mine << shift_;
  }
  // local slot -> global vector index (may be >= nvec in the last, partial block)
  __host__ __device__ __forceinline__ size_t global(size_t slot) const {
    const size_t q = slot >> shift, w = slot & (((size_t)1 << shift) - 1);
    return ((q * n + rank) << shift) + w;
  }
};

// `unrolled` over this rank's local slots, CTA bid of nb working on them: each thread loads the
// vectors g < own.nvec of UNROLL slots (load(g, v)) before it stores any of them (store(g, v)).
// twoshot_body, scan_kernel and nvls_body keep this loop written out: through the helper they
// compiled to different SASS.
template <int UNROLL, typename V, typename Load, typename Store>
__device__ __forceinline__ void unrolled_owned(const Owner& own, unsigned bid, unsigned nb, Load load, Store store) {
  const size_t step = (size_t)nb * blockDim.x * UNROLL;
  for (size_t l0 = (size_t)bid * blockDim.x * UNROLL + threadIdx.x; l0 < own.slots; l0 += step) {
    V v[UNROLL];
    size_t gi[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t l = l0 + (size_t)u * blockDim.x;
      gi[u] = l < own.slots ? own.global(l) : own.nvec;
      if (gi[u] < own.nvec) load(gi[u], v[u]);
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u)
      if (gi[u] < own.nvec) store(gi[u], v[u]);
  }
}

// ---------------------------------------------------------------------------------------------
// Allreduce, two-shot fused in one pass: the owner of a vector loads it from all n ranks
// (7 concurrent NVLink read streams + 1 local), reduces in rank order and stores the result into
// every rank's recv buffer (7 NVLink write streams + 1 local).  Reduce-scatter and all-gather
// traffic therefore overlap in both link directions and no mid barrier is needed.
// In place is safe: a vector is read and then written only by its owner.
// ---------------------------------------------------------------------------------------------
// bid / nb: this CTA's index and the number of CTAs working on the message (a fused kernel may give
// only part of its grid to this body).  only_dst >= 0: the reduced value is stored into that
// rank's recv buffer only (Reduce); -1: into every rank's (Allreduce).
template <typename T, typename Op, int NR, int UNROLL>
__device__ __forceinline__ void twoshot_body(const Comm& c, const uint64_t* s_a, const uint64_t* s_b, size_t count, uint32_t shift,
                                             unsigned bid, unsigned nb, int only_dst = -1) {
  const int n = NR ? NR : c.n;
  constexpr int R = NR ? NR : kMaxRanks;
  constexpr int EPV = Pack<T>::N;
  const size_t tid = threadIdx.x;
  if (all_aligned16(s_a, s_b, n)) {
    const size_t nvec = count / EPV;
    const Owner own(nvec, shift, n, c.rank);
    // base pointers live in shared memory, not in 2 x R registers per thread (ptxas spilled the
    // 8-rank and generic instances with register arrays)
    __shared__ const char* src[kMaxRanks];
    __shared__ char* dst[kMaxRanks];
    if (tid < (size_t)R) {
      const int r = (int)tid;
      const int q = r < n ? r : 0;
      src[r] = c.base[q] + s_a[q];
      // stores start at the next rank so the ranks do not all hit the same target at once
      const int w = only_dst >= 0 ? only_dst : (c.rank + 1 + r) % n;
      dst[r] = c.base[w] + s_b[w];
    }
    __syncthreads();
    const int ndst = only_dst >= 0 ? 1 : n;
    const size_t step = (size_t)nb * blockDim.x * UNROLL;
    for (size_t l0 = (size_t)bid * blockDim.x * UNROLL + tid; l0 < own.slots; l0 += step) {
      Pack<T> v[UNROLL][R];
      size_t gi[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const size_t l = l0 + (size_t)u * blockDim.x;
        gi[u] = l < own.slots ? own.global(l) : nvec;
        if (gi[u] < nvec) {
#pragma unroll
          for (int r = 0; r < R; ++r)
            if (r < n) v[u][r] = ld_pack<T>(src[r] + gi[u] * 16);
        }
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        if (gi[u] < nvec) {
          Pack<T> acc = v[u][0];
#pragma unroll
          for (int r = 1; r < R; ++r)
            if (r < n) acc = combine<T, Op>(acc, v[u][r]);
#pragma unroll
          for (int r = 0; r < R; ++r)
            if (r < ndst) st_pack<T>(dst[r] + gi[u] * 16, acc);
        }
      }
    }
    // elements past the last whole vector: reduced and pushed by the last rank
    if (c.rank == n - 1) reduce_store_elements<T, Op>(c, s_a, s_b, n, nvec * EPV, count, bid, nb, only_dst);
  } else {
    // unaligned buffers: contiguous ownership by element, scalar accesses
    const Range mine = owned_elements(count, n, c.rank);
    reduce_store_elements<T, Op>(c, s_a, s_b, n, mine.lo, mine.hi, bid, nb, only_dst);
  }
}

template <typename T, typename Op, int NR, int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
allreduce_twoshot_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t count, uint32_t shift, int only_dst) {
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    twoshot_body<T, Op, NR, UNROLL>(c, s_a, s_b, count, shift, blockIdx.x, gridDim.x, only_dst);
  });
}

// ---------------------------------------------------------------------------------------------
// Scan / Exscan: prefix reductions in rank order.  Rank r receives ((x_0 op x_1) op ...) op x_r
// (Scan) or the same up to x_{r-1} (Exscan; rank 0 receives nothing).  Same ownership and traffic
// as the two-shot Allreduce: the owner of a vector loads it from every rank's send (Exscan never
// needs rank n-1's), forms the running prefix in registers and stores prefix r (r-1) into rank r's
// recv, starting at the next rank.  In place is safe for the same reason as in two-shot.  Under
// Exscan rank 0 announces its send offset as its recv, and nothing is ever stored to rank 0.
// ---------------------------------------------------------------------------------------------
// One element e, scalar, in rank order: the unaligned body and the tail past the last whole vector.
// Rank r's input is loaded before rank r's recv is stored, so in place holds here too.
template <typename T, typename Op, bool EXCLUSIVE>
__device__ __forceinline__ void scan_element(const Comm& c, const uint64_t* s_a, const uint64_t* s_b, int n, size_t e) {
  auto in = [&](int r) { return reinterpret_cast<const volatile T*>(c.base[r] + s_a[r])[e]; };
  auto out = [&](int r, T v) { reinterpret_cast<volatile T*>(c.base[r] + s_b[r])[e] = v; };
  T acc = in(0);
  if (!EXCLUSIVE) out(0, acc);
  for (int r = 1; r < n; ++r) {
    if (EXCLUSIVE) {
      const T x = r < n - 1 ? in(r) : T(0);
      out(r, acc);
      if (r < n - 1) acc = Op::template apply<T>(acc, x);
    } else {
      acc = Op::template apply<T>(acc, in(r));
      out(r, acc);
    }
  }
}

template <typename T, typename Op, int NR, int UNROLL, bool EXCLUSIVE>
__global__ void __launch_bounds__(kThreads, 1)
scan_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t count, uint32_t shift) {
  __shared__ const char* src[kMaxRanks];
  __shared__ char* dst[kMaxRanks];
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    const int n = NR ? NR : c.n;
    const int nin = EXCLUSIVE ? n - 1 : n; // ranks whose input any result needs
    constexpr int R = NR ? NR : kMaxRanks;
    constexpr int EPV = Pack<T>::N;
    const size_t tid = threadIdx.x;
    const size_t nthreads = (size_t)gridDim.x * blockDim.x;
    if (all_aligned16(s_a, s_b, n)) {
      const size_t nvec = count / EPV;
      const Owner own(nvec, shift, n, c.rank);
      if (tid < (size_t)R) {
        const int r = (int)tid < n ? (int)tid : 0;
        src[tid] = c.base[r] + s_a[r];
        dst[tid] = c.base[r] + s_b[r];
      }
      __syncthreads();
      const size_t step = nthreads * UNROLL;
      for (size_t l0 = (size_t)blockIdx.x * blockDim.x * UNROLL + tid; l0 < own.slots; l0 += step) {
        Pack<T> v[UNROLL][R];
        size_t gi[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
          const size_t l = l0 + (size_t)u * blockDim.x;
          gi[u] = l < own.slots ? own.global(l) : nvec;
          if (gi[u] < nvec) {
#pragma unroll
            for (int r = 0; r < R; ++r)
              if (r < nin) v[u][r] = ld_pack<T>(src[r] + gi[u] * 16);
          }
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
          if (gi[u] < nvec) {
#pragma unroll
            for (int r = 1; r < R; ++r) // v[u][r] becomes prefix r
              if (r < nin) v[u][r] = combine<T, Op>(v[u][r - 1], v[u][r]);
            // rank r's result is prefix r (Scan) or prefix r-1 (Exscan); ranks after this one first
#pragma unroll
            for (int r = EXCLUSIVE ? 1 : 0; r < R; ++r)
              if (r > c.rank && r < n) st_pack<T>(dst[r] + gi[u] * 16, v[u][EXCLUSIVE ? r - 1 : r]);
#pragma unroll
            for (int r = EXCLUSIVE ? 1 : 0; r < R; ++r)
              if (r <= c.rank) st_pack<T>(dst[r] + gi[u] * 16, v[u][EXCLUSIVE ? r - 1 : r]);
          }
        }
      }
      // elements past the last whole vector: reduced and pushed by the last rank
      if (c.rank == n - 1)
        for (size_t e = nvec * EPV + (size_t)blockIdx.x * blockDim.x + tid; e < count; e += nthreads) scan_element<T, Op, EXCLUSIVE>(c, s_a, s_b, n, e);
    } else {
      // unaligned buffers: contiguous ownership by element, scalar accesses
      const Range mine = owned_elements(count, n, c.rank);
      for (size_t e = mine.lo + (size_t)blockIdx.x * blockDim.x + tid; e < mine.hi; e += nthreads) scan_element<T, Op, EXCLUSIVE>(c, s_a, s_b, n, e);
    }
  });
}

// ---------------------------------------------------------------------------------------------
// Allreduce, two-shot with shared-memory staging (TMA bulk copies).  Same ownership, traffic and
// rank-order arithmetic as allreduce_twoshot_kernel, but the SM's load/store units never touch
// NVLink: one producer thread per CTA streams kChunk-byte tiles of slice j from all NR heaps into
// a ring of shared-memory stages with cp.async.bulk (completion on an mbarrier); 8 consumer warps
// reduce the NR tiles out of shared memory into an output tile, and one thread writes that tile
// to all NR recv buffers with cp.async.bulk shared->global.  In flight per SM: kStages*NR*kChunk.
// ---------------------------------------------------------------------------------------------
constexpr int kSmemChunk = 4096;       // bytes per tile per rank (256 consumer threads x 16 B)
constexpr int kSmemStages = 4;
constexpr int kSmemOutStages = 2;
constexpr int kSmemConsumers = 256;
constexpr int kSmemThreads = kSmemConsumers + 32;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

template <typename T, typename Op, int NR>
__global__ void __launch_bounds__(kSmemThreads, 1)
allreduce_twoshot_smem_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t count, uint32_t shift) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kSmemStages], empty_bar[kSmemStages];
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    unsigned char* in_tiles = smem_raw;                                         // [stage][rank][chunk]
    unsigned char* out_tiles = smem_raw + (size_t)kSmemStages * NR * kSmemChunk; // [ostage][chunk]
    constexpr int EPV = Pack<T>::N;
    const int tid = threadIdx.x;
    const bool al = all_aligned16(s_a, s_b, NR);
    const size_t nvec = al ? count / EPV : 0;
    // shift >= 8 (a block is a whole number of 4 KiB tiles); tile t covers local slots [t*256, t*256+256)
    const Owner own(nvec, shift, NR, c.rank);
    constexpr size_t kTileVecs = kSmemChunk / 16;
    const size_t ntiles = own.slots / kTileVecs;
    if (tid == 0) {
      for (int s = 0; s < kSmemStages; ++s) {
        mbar_init(&full_bar[s], 1);
        mbar_init(&empty_bar[s], kSmemConsumers / 32);
      }
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid >= kSmemConsumers) {
      // ---- producer warp: one lane drives the TMA loads ----
      if (tid == kSmemConsumers) {
        uint32_t it = 0;
        for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
          if (own.global(t * kTileVecs) >= nvec) continue;
          const int s = it % kSmemStages;
          const uint32_t use = it / kSmemStages;
          ++it;
          if (use > 0) mbar_wait(&empty_bar[s], (use - 1) & 1);
          const size_t g0 = own.global(t * kTileVecs);
          const size_t off = g0 * 16;
          const uint32_t bytes = (uint32_t)((nvec - g0) < kTileVecs ? (nvec - g0) * 16 : (size_t)kSmemChunk);
          mbar_expect_tx(&full_bar[s], bytes * NR);
#pragma unroll
          for (int r = 0; r < NR; ++r)
            bulk_g2s(in_tiles + ((size_t)s * NR + r) * kSmemChunk, c.base[r] + s_a[r] + off, bytes, &full_bar[s]);
        }
      }
    } else {
      // ---- consumer warps ----
      uint32_t nit = 0;
      for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const size_t g0 = own.global(t * kTileVecs);
        if (g0 >= nvec) continue;
        const uint32_t it = nit++;
        const int s = it % kSmemStages;
        const int os = it % kSmemOutStages;
        const uint32_t bytes = (uint32_t)((nvec - g0) < kTileVecs ? (nvec - g0) * 16 : (size_t)kSmemChunk);
        mbar_wait(&full_bar[s], (it / kSmemStages) & 1);
        if (it >= (uint32_t)kSmemOutStages) { // the stores that read out_tiles[os] two tiles ago must have drained it
          if (tid == 0) bulk_wait_read<kSmemOutStages - 1>();
          asm volatile("bar.sync 1, %0;" ::"n"(kSmemConsumers) : "memory");
        }
        if ((uint32_t)tid * 16 < bytes) {
          const unsigned char* src = in_tiles + (size_t)s * NR * kSmemChunk + (size_t)tid * 16;
          Pack<T> acc = *reinterpret_cast<const Pack<T>*>(src);
#pragma unroll
          for (int r = 1; r < NR; ++r) acc = combine<T, Op>(acc, *reinterpret_cast<const Pack<T>*>(src + (size_t)r * kSmemChunk));
          *reinterpret_cast<Pack<T>*>(out_tiles + (size_t)os * kSmemChunk + (size_t)tid * 16) = acc;
        }
        fence_proxy_async_smem(); // generic-proxy writes to out_tiles -> visible to the bulk-copy engine
        asm volatile("bar.sync 1, %0;" ::"n"(kSmemConsumers) : "memory");
        if ((tid & 31) == 0) mbar_arrive(&empty_bar[s]); // this warp is done reading in_tiles[s]
        if (tid == 0) {
          const size_t off = g0 * 16;
#pragma unroll
          for (int r = 0; r < NR; ++r) {
            const int w = (c.rank + 1 + r) % NR;
            bulk_s2g(c.base[w] + s_b[w] + off, out_tiles + (size_t)os * kSmemChunk, bytes);
          }
          bulk_commit();
        }
      }
      if (tid == 0) bulk_wait<0>(); // every peer write of this CTA has been performed
    }
    // elements outside whole 16-byte vectors, or everything when unaligned: scalar, last rank / by ownership
    // (stored here, not through reduce_store_elements, which compiled to different SASS in this kernel)
    const size_t gtid = (size_t)blockIdx.x * blockDim.x + tid;
    const size_t gstride = (size_t)gridDim.x * blockDim.x;
    const Range scalar = al ? Range{c.rank == NR - 1 ? nvec * EPV : count, count} : owned_elements(count, NR, c.rank);
    for (size_t e = scalar.lo + gtid; e < scalar.hi; e += gstride) {
      const T acc = reduce_ranks<T, Op>(c, s_a, NR, e);
      for (int r = 0; r < NR; ++r) reinterpret_cast<volatile T*>(c.base[r] + s_b[r])[e] = acc;
    }
  });
}

// ---------------------------------------------------------------------------------------------
// Allreduce, ring: n-1 reduce-scatter steps then n-1 all-gather steps; each rank only ever loads
// from its predecessor.  CTA b of rank r depends only on CTA b of rank r-1 (same vector subset on
// every rank), signalled through ring[b] in the successor's heap.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t* ring_flag(const Comm& c, int owner, int block) {
  return reinterpret_cast<uint32_t*>(c.base[owner] + kRingFlagsOff) + block;
}

template <typename T, typename Op>
__global__ void __launch_bounds__(kThreads, 1)
allreduce_ring_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t count) {
  __shared__ uint64_t s_a[kMaxRanks], s_b[kMaxRanks];
  const bool call_ok = sync_start(c, send_off, recv_off, s_a, s_b);
  if (!call_ok) { // ranks disagree about this call: touch nothing, leave through the end barrier
    sync_end_failed(c);
    return;
  }
  const int n = c.n, r = c.rank;
  const int prev = (r + n - 1) % n, next = (r + 1) % n;
  constexpr int EPV = Pack<T>::N;
  const bool al = all_aligned16(s_a, s_b, n);
  // Chunks are made of whole 16-byte groups whatever the alignment, so the summation order is a
  // function of (count, n, dtype) only; the count % EPV tail is reduced in rank order.
  const size_t groups = count / EPV;
  const size_t per = (groups + n - 1) / n;
  const char* my_send = c.base[r] + s_a[r];
  char* my_recv = c.base[r] + s_b[r];
  const char* prev_send = c.base[prev] + s_a[prev];
  const char* prev_recv = c.base[prev] + s_b[prev];
  const uint32_t fbase = c.epoch * 8u;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const int steps = 2 * (n - 1);
  for (int g = 0; g < steps; ++g) {
    const bool rs = g < n - 1;
    const int s = rs ? g : g - (n - 1);
    const int chunk = rs ? (r - s - 1 + 2 * n) % n : (r - s + 2 * n) % n;
    if (g > 0) {
      if (threadIdx.x == 0) wait_flag(ring_flag(c, r, blockIdx.x), fbase + (uint32_t)g, c);
      __syncthreads();
    }
    // owned_elements(groups, n, chunk), written out: through the helper this kernel compiled to different SASS
    const size_t lo = per * chunk < groups ? per * chunk : groups;
    const size_t hi = lo + per < groups ? lo + per : groups;
    const char* in = (g == 0) ? prev_send : prev_recv;
    if (al) {
      for (size_t i = lo + tid; i < hi; i += stride) {
        Pack<T> p = ld_pack_sys<T>(in + i * 16);
        if (rs) {
          Pack<T> m = ld_pack<T>(my_send + i * 16);
          p = combine<T, Op>(p, m);
        }
        st_pack<T>(my_recv + i * 16, p);
      }
    } else {
      for (size_t e = lo * EPV + tid; e < hi * EPV; e += stride) {
        T p = reinterpret_cast<const volatile T*>(in)[e];
        if (rs) p = Op::template apply<T>(p, reinterpret_cast<const volatile T*>(my_send)[e]);
        reinterpret_cast<volatile T*>(my_recv)[e] = p;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) st_release_sys(ring_flag(c, next, blockIdx.x), fbase + (uint32_t)g + 1u);
  }
  // tail: at most EPV-1 elements, one per thread of CTA 0, kept in a register across the barrier
  const size_t te = groups * EPV + tid;
  T tail = T(0);
  if (te < count) tail = reduce_ranks<T, Op>(c, s_a, n, te);
  sync_end(c);
  __syncthreads(); // sync_end's waits are done by threads 0..n-1 only
  // after the barrier nobody reads this rank's send buffer any more (in-place safe)
  if (te < count) reinterpret_cast<T*>(my_recv)[te] = tail;
}

// ---------------------------------------------------------------------------------------------
// Allreduce through the switch (NVLS): rank j reduces slice j with multimem.ld_reduce (the
// NVSwitch fetches the slice from all n heaps and returns the reduced value) and multicasts the
// result into every rank's recv buffer with multimem.st.  Needs every rank to use the same heap
// offsets (checked after sync_start; otherwise falls back to the two-shot body by returning 0).
// ---------------------------------------------------------------------------------------------
template <typename T, typename Op> struct Multimem;
template <> struct Multimem<float, OpSum> {
  __device__ __forceinline__ static Pack<float> ld_reduce(const void* p) {
    Pack<float> r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.v[0]), "=f"(r.v[1]), "=f"(r.v[2]), "=f"(r.v[3]) : "l"(p) : "memory");
    return r;
  }
};
template <> struct Multimem<double, OpSum> {
  __device__ __forceinline__ static Pack<double> ld_reduce(const void* p) {
    Pack<double> r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.f64 %0, [%1];" : "=d"(r.v[0]) : "l"(p) : "memory");
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.f64 %0, [%1];" : "=d"(r.v[1]) : "l"((const char*)p + 8) : "memory");
    return r;
  }
};
template <> struct Multimem<long long, OpSum> {
  __device__ __forceinline__ static Pack<long long> ld_reduce(const void* p) {
    Pack<long long> r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.u64 %0, [%1];" : "=l"(r.v[0]) : "l"(p) : "memory");
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.u64 %0, [%1];" : "=l"(r.v[1]) : "l"((const char*)p + 8) : "memory");
    return r;
  }
};
template <> struct Multimem<long long, OpMax> {
  __device__ __forceinline__ static Pack<long long> ld_reduce(const void* p) {
    Pack<long long> r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.max.s64 %0, [%1];" : "=l"(r.v[0]) : "l"(p) : "memory");
    asm volatile("multimem.ld_reduce.relaxed.sys.global.max.s64 %0, [%1];" : "=l"(r.v[1]) : "l"((const char*)p + 8) : "memory");
    return r;
  }
};
template <> struct Multimem<long long, OpMin> {
  __device__ __forceinline__ static Pack<long long> ld_reduce(const void* p) {
    Pack<long long> r;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.min.s64 %0, [%1];" : "=l"(r.v[0]) : "l"(p) : "memory");
    asm volatile("multimem.ld_reduce.relaxed.sys.global.min.s64 %0, [%1];" : "=l"(r.v[1]) : "l"((const char*)p + 8) : "memory");
    return r;
  }
};
__device__ __forceinline__ void multimem_st16(void* p, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p),
               "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)),
               "f"(__uint_as_float(v.w))
               : "memory");
}

// The switch part of a message: vectors [0, nvec) of the buffers at heap offsets send_off /
// recv_off (the same on every rank).  only_dst < 0: the reduced vector is multicast into every
// rank's recv buffer; >= 0: stored into that rank's recv buffer only (Reduce).
template <typename T, typename Op, int UNROLL>
__device__ __forceinline__ void nvls_body(const Comm& c, uint64_t send_off, uint64_t recv_off, size_t nvec, uint32_t shift,
                                          unsigned bid, unsigned nb, int only_dst = -1) {
  const Owner own(nvec, shift, c.n, c.rank);
  const char* src = c.mc + send_off;
  char* dst = only_dst < 0 ? c.mc + recv_off : c.base[only_dst] + recv_off;
  const size_t tid = threadIdx.x;
  const size_t step = (size_t)nb * blockDim.x * UNROLL;
  for (size_t l0 = (size_t)bid * blockDim.x * UNROLL + tid; l0 < own.slots; l0 += step) {
    Pack<T> v[UNROLL];
    size_t gi[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t l = l0 + (size_t)u * blockDim.x;
      gi[u] = l < own.slots ? own.global(l) : nvec;
      if (gi[u] < nvec) v[u] = Multimem<T, Op>::ld_reduce(src + gi[u] * 16);
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      if (gi[u] < nvec) {
        union { uint4 u4; Pack<T> k; } x;
        x.k = v[u];
        if (only_dst < 0) multimem_st16(dst + gi[u] * 16, x.u4);
        else stg16(dst + gi[u] * 16, x.u4);
      }
    }
  }
}

__device__ __forceinline__ bool symmetric_offsets(const uint64_t* s_a, const uint64_t* s_b, uint64_t send_off, uint64_t recv_off, int n) {
  bool sym = ((send_off | recv_off) & 15) == 0;
  for (int r = 0; r < n; ++r) sym = sym && s_a[r] == send_off && s_b[r] == recv_off;
  return sym;
}

template <typename T, typename Op, int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
allreduce_nvls_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t count, uint32_t shift, int only_dst) {
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    constexpr int EPV = Pack<T>::N;
    // Reduce (only_dst >= 0): recv matters on the root only; the other ranks' recv offsets are ignored
    bool symmetric;
    if (only_dst < 0) symmetric = symmetric_offsets(s_a, s_b, send_off, recv_off, c.n);
    else {
      symmetric = ((send_off | s_b[only_dst]) & 15) == 0;
      for (int r = 0; r < c.n; ++r) symmetric = symmetric && s_a[r] == send_off;
    }
    if (symmetric) {
      const size_t nvec = count / EPV;
      nvls_body<T, Op, UNROLL>(c, send_off, only_dst < 0 ? recv_off : s_b[only_dst], nvec, shift, blockIdx.x, gridDim.x, only_dst);
      // count % EPV trailing elements: last rank, rank order, P2P
      if (c.rank == c.n - 1) reduce_store_elements<T, Op>(c, s_a, s_b, c.n, nvec * EPV, count, blockIdx.x, gridDim.x, only_dst);
    } else {
      // the multicast address needs the same offsets on every rank; otherwise the P2P two-shot body
      twoshot_body<T, Op, 0, 1>(c, s_a, s_b, count, shift, blockIdx.x, gridDim.x, only_dst);
    }
  });
}

// ---------------------------------------------------------------------------------------------
// Allreduce, hybrid: for when the switch reduction (multimem) saturates below the link rate, so a
// part of the message goes the P2P way at the same time: CTAs [0, nb_nvls) run nvls_body on
// vectors [0, split), the remaining CTAs run the fused P2P two-shot body on [split, nvec) and the
// tail.  Every element is still reduced exactly once by its owner and the same bits reach every
// rank.  split and nb_nvls are functions of (count, n, tuning parameters) only.
// ---------------------------------------------------------------------------------------------
template <typename T, typename Op, int NR, int UN, int UP>
__global__ void __launch_bounds__(kThreads, 1)
allreduce_hybrid_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t count, uint32_t shift_nvls, uint32_t shift_p2p,
                        size_t split_vec, unsigned nb_nvls) {
  __shared__ uint64_t s_a2[kMaxRanks], s_b2[kMaxRanks];
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    constexpr int EPV = Pack<T>::N;
    if (symmetric_offsets(s_a, s_b, send_off, recv_off, c.n)) {
      if (blockIdx.x < nb_nvls) {
        nvls_body<T, Op, UN>(c, send_off, recv_off, split_vec, shift_nvls, blockIdx.x, nb_nvls);
      } else {
        if (threadIdx.x < (unsigned)c.n) {
          s_a2[threadIdx.x] = s_a[threadIdx.x] + split_vec * 16;
          s_b2[threadIdx.x] = s_b[threadIdx.x] + split_vec * 16;
        }
        __syncthreads();
        twoshot_body<T, Op, NR, UP>(c, s_a2, s_b2, count - split_vec * EPV, shift_p2p, blockIdx.x - nb_nvls, gridDim.x - nb_nvls);
      }
    } else {
      twoshot_body<T, Op, NR, UP>(c, s_a, s_b, count, shift_p2p, blockIdx.x, gridDim.x);
    }
  });
}

// ---------------------------------------------------------------------------------------------
// ReduceScatter: rank j ends up with op over r of block j of rank r's send buffer (n blocks of
// `count` elements), in rank order.  Only the owner reads block j, so recv may alias the owner's
// own block of send.  P2P form: n concurrent read streams.  NVLS form: multimem.ld_reduce.
// This is the first half of the two-shot allreduce exposed on its own.
// ---------------------------------------------------------------------------------------------
template <typename T, typename Op, int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
reduce_scatter_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t count) {
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t*) {
    __shared__ const char* src[kMaxRanks];
    const int n = c.n;
    constexpr int EPV = Pack<T>::N;
    const size_t blk_bytes = count * sizeof(T);
    if (threadIdx.x < (unsigned)n) src[threadIdx.x] = c.base[threadIdx.x] + s_a[threadIdx.x] + (size_t)c.rank * blk_bytes;
    __syncthreads();
    char* out = c.base[c.rank] + recv_off;
    uint64_t m = recv_off | blk_bytes; // block j of every rank must be 16-byte aligned for the vector path
    for (int r = 0; r < n; ++r) m |= s_a[r];
    const size_t nvec = (m & 15) == 0 ? count / EPV : 0;
    unrolled<UNROLL, Pack<T>>(
        0, nvec,
        [&](size_t i, Pack<T>& acc) {
          acc = ld_pack<T>(src[0] + i * 16);
          for (int r = 1; r < n; ++r) acc = combine<T, Op>(acc, ld_pack<T>(src[r] + i * 16));
        },
        [&](size_t i, const Pack<T>& acc) { st_pack<T>(out + i * 16, acc); });
    for (size_t e = nvec * EPV + (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < count; e += (size_t)gridDim.x * blockDim.x)
      reinterpret_cast<T*>(out)[e] = reduce_ranks<T, Op>([&](int r) { return src[r]; }, n, e);
  });
}

template <typename T, typename Op, int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
reduce_scatter_nvls_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t count) {
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    const int n = c.n;
    constexpr int EPV = Pack<T>::N;
    const size_t blk_bytes = count * sizeof(T);
    bool symmetric = ((send_off | recv_off | blk_bytes) & 15) == 0;
    for (int r = 0; r < n; ++r) symmetric = symmetric && s_a[r] == send_off && (s_b[r] & 15) == 0;
    char* out = c.base[c.rank] + recv_off;
    const size_t tid = threadIdx.x;
    if (symmetric) {
      const char* src = c.mc + send_off + (size_t)c.rank * blk_bytes;
      // written out: through `unrolled` this loop compiled to different SASS (+1 register for f64)
      const size_t nvec = count / EPV; // blk_bytes % 16 == 0: no tail
      const size_t step = (size_t)gridDim.x * blockDim.x * UNROLL;
      for (size_t i0 = (size_t)blockIdx.x * blockDim.x * UNROLL + tid; i0 < nvec; i0 += step) {
        Pack<T> v[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
          const size_t i = i0 + (size_t)u * blockDim.x;
          if (i < nvec) v[u] = Multimem<T, Op>::ld_reduce(src + i * 16);
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
          const size_t i = i0 + (size_t)u * blockDim.x;
          if (i < nvec) st_pack<T>(out + i * 16, v[u]);
        }
      }
    } else { // P2P, scalar, rank order (every rank takes this branch: the decision uses exchanged offsets only)
      for (size_t e = (size_t)blockIdx.x * blockDim.x + tid; e < count; e += (size_t)gridDim.x * blockDim.x)
        reinterpret_cast<T*>(out)[e] = reduce_ranks<T, Op>([&](int r) { return c.base[r] + s_a[r] + (size_t)c.rank * blk_bytes; }, n, e);
    }
  });
}

// Coherent (system-scope) loads of one access unit, for data that a peer rewrites during the
// same kernel (ring steps): never served from a stale L1 line.
__device__ __forceinline__ uint4 ld_unit_sys(const volatile uint4* p) { return ldg16_sys((const void*)p); }
__device__ __forceinline__ unsigned long long ld_unit_sys(const volatile unsigned long long* p) { return *p; }
__device__ __forceinline__ unsigned int ld_unit_sys(const volatile unsigned int* p) { return *p; }
__device__ __forceinline__ unsigned char ld_unit_sys(const volatile unsigned char* p) { return *p; }

// ---------------------------------------------------------------------------------------------
// Allgather / Bcast bodies.  U is the access unit the host picked from ITS offsets and the size;
// after sync_start every rank's offsets are known, and a rank that sees a less aligned peer
// drops to the byte-wide instance of the same body.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool all_aligned_to(const uint64_t* s_a, const uint64_t* s_b, int n, unsigned unit) {
  uint64_t m = 0;
  for (int r = 0; r < n; ++r) m |= s_a[r] | s_b[r];
  return (m & (unit - 1)) == 0;
}

// Runs body(unit, unroll) with the host's unit U and UNROLL when every rank's offsets allow U
// (`aligned`, typically all_aligned_to), else with bytes and an unroll of 1.  `unit` is a value of
// the unit type and `unroll` a std::integral_constant, so the body names them as decltype(unit)
// and unroll.
template <typename U, int UNROLL, typename Body>
__device__ __forceinline__ void unit_or_bytes(bool aligned, Body body) {
  if (sizeof(U) == 1 || aligned) body(U{}, std::integral_constant<int, UNROLL>{});
  else body((unsigned char)0, std::integral_constant<int, 1>{});
}

// The copy loop of the push and pull bodies: units [lo, hi) of src, grid-strided, UNROLL loads in
// flight per thread, then each unit stored to the first `ntargets` of dst[0..MAXT).  Written out
// rather than built on `unrolled`, which changed the SASS of allgather_push_kernel and
// bcast_nvls_kernel.
template <typename U, int UNROLL, int MAXT>
__device__ __forceinline__ void copy_units(const U* src, U* const* dst, int ntargets, size_t lo, size_t hi) {
  const size_t step = (size_t)gridDim.x * blockDim.x * UNROLL;
  for (size_t i0 = lo + (size_t)blockIdx.x * blockDim.x * UNROLL + threadIdx.x; i0 < hi; i0 += step) {
    U v[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t i = i0 + (size_t)u * blockDim.x;
      if (i < hi) v[u] = src[i];
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t i = i0 + (size_t)u * blockDim.x;
      if (i < hi) {
#pragma unroll
        for (int r = 0; r < MAXT; ++r)
          if (r < ntargets) dst[r][i] = v[u];
      }
    }
  }
}

// Direct push: every rank streams its block [lo, lo + bytes) once from local HBM and stores it at lo
// in the recv buffer of `only_dst` (Gather) or of all n ranks, own last (only_dst == -1: Allgather,
// Allgatherv).  The own copy is skipped when the call is in place (send == recv + lo).
template <typename U, int UNROLL>
__device__ __forceinline__ void push_block_body(const Comm& c, const uint64_t* s_a, const uint64_t* s_b, uint64_t lo,
                                                uint64_t bytes, int only_dst) {
  const int n = c.n;
  const size_t units = bytes / sizeof(U);
  const U* src = reinterpret_cast<const U*>(c.base[c.rank] + s_a[c.rank]);
  const bool inplace = s_a[c.rank] == s_b[c.rank] + lo;
  U* dst[kMaxRanks];
#pragma unroll
  for (int r = 0; r < kMaxRanks; ++r) {
    const int w = only_dst >= 0 ? only_dst : (c.rank + 1 + r) % n; // w == rank when r == n-1
    dst[r] = reinterpret_cast<U*>(c.base[w] + s_b[w] + lo);
  }
  const int ntargets = only_dst >= 0 ? (only_dst == c.rank && inplace ? 0 : 1) : (inplace ? n - 1 : n);
  copy_units<U, UNROLL, kMaxRanks>(src, dst, ntargets, 0, units);
}

// push_block_body with lo = rank * bytes_per_rank and every rank a target, for the P2P fallback of
// allgather_nvls_kernel: with push_block_body that kernel compiled to 64 registers and 56 more
// instructions than with this body.
template <typename U, int UNROLL>
__device__ __forceinline__ void allgather_push_body(const Comm& c, const uint64_t* s_a, const uint64_t* s_b,
                                                    size_t bytes_per_rank) {
  const int n = c.n;
  const size_t units = bytes_per_rank / sizeof(U);
  const U* src = reinterpret_cast<const U*>(c.base[c.rank] + s_a[c.rank]);
  const bool inplace = s_a[c.rank] == s_b[c.rank] + (uint64_t)c.rank * bytes_per_rank;
  U* dst[kMaxRanks];
#pragma unroll
  for (int r = 0; r < kMaxRanks; ++r) {
    const int w = (c.rank + 1 + r) % n; // w == rank when r == n-1
    dst[r] = reinterpret_cast<U*>(c.base[w] + s_b[w] + (size_t)c.rank * bytes_per_rank);
  }
  copy_units<U, UNROLL, kMaxRanks>(src, dst, inplace ? n - 1 : n, 0, units);
}

template <typename U, int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
allgather_push_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t bytes_per_rank) {
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    unit_or_bytes<U, UNROLL>(all_aligned_to(s_a, s_b, c.n, sizeof(U)), [&](auto unit, auto unroll) {
      push_block_body<decltype(unit), unroll>(c, s_a, s_b, (uint64_t)c.rank * bytes_per_rank, bytes_per_rank, -1);
    });
  });
}

// Ring allgather: step s pulls block (r - s - 1) from the predecessor.
template <typename U>
__device__ __forceinline__ void allgather_ring_body(const Comm& c, const uint64_t* s_a, const uint64_t* s_b,
                                                    size_t bytes_per_rank) {
  const int n = c.n, r = c.rank;
  const int prev = (r + n - 1) % n, next = (r + 1) % n;
  const size_t units = bytes_per_rank / sizeof(U);
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  char* my_recv = c.base[r] + s_b[r];
  const uint32_t fbase = c.epoch * 8u;
  if (s_a[r] != s_b[r] + (uint64_t)r * bytes_per_rank) { // own block, out of place
    const U* s = reinterpret_cast<const U*>(c.base[r] + s_a[r]);
    U* d = reinterpret_cast<U*>(my_recv + (size_t)r * bytes_per_rank);
    for (size_t i = tid; i < units; i += stride) d[i] = s[i];
  }
  for (int s = 0; s < n - 1; ++s) {
    const int blk = (r - s - 1 + 2 * n) % n;
    if (s > 0) {
      if (threadIdx.x == 0) wait_flag(ring_flag(c, r, blockIdx.x), fbase + (uint32_t)s, c);
      __syncthreads();
    }
    const volatile U* in = (s == 0) ? reinterpret_cast<const volatile U*>(c.base[prev] + s_a[prev])
                                    : reinterpret_cast<const volatile U*>(c.base[prev] + s_b[prev] + (size_t)blk * bytes_per_rank);
    U* out = reinterpret_cast<U*>(my_recv + (size_t)blk * bytes_per_rank);
    for (size_t i = tid; i < units; i += stride) out[i] = ld_unit_sys(in + i);
    __syncthreads();
    if (threadIdx.x == 0) st_release_sys(ring_flag(c, next, blockIdx.x), fbase + (uint32_t)s + 1u);
  }
}

template <typename U>
__global__ void __launch_bounds__(kThreads, 1)
allgather_ring_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t bytes_per_rank) {
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    unit_or_bytes<U, 1>(all_aligned_to(s_a, s_b, c.n, sizeof(U)), [&](auto unit, auto) {
      allgather_ring_body<decltype(unit)>(c, s_a, s_b, bytes_per_rank);
    });
  });
}

// ---------------------------------------------------------------------------------------------
// Bcast
// ---------------------------------------------------------------------------------------------
// mode 0 (one-shot): every non-root pulls the whole buffer from root (root egress (n-1)*S).
// mode 1 (two-shot, fused): non-root k pulls slice k from root and stores it locally and into
// the other non-roots, so root sends every byte once and all links run in both directions.
template <typename U, int UNROLL>
__device__ __forceinline__ void bcast_body(const Comm& c, const uint64_t* s_a, size_t bytes, int root, int mode) {
  const int n = c.n;
  if (c.rank == root) return;
  const size_t units = bytes / sizeof(U);
  const U* src = reinterpret_cast<const U*>(c.base[root] + s_a[root]);
  size_t lo = 0, hi = units;
  int ntargets = 1;
  U* dst[kMaxRanks];
  dst[0] = reinterpret_cast<U*>(c.base[c.rank] + s_a[c.rank]);
  if (mode == 1) {
    // slices are cut in bytes on 16-byte granules so that ranks running different access widths
    // (their offsets differ in alignment) still cover the buffer exactly once
    const int m = n - 1;
    const int k = c.rank < root ? c.rank : c.rank - 1;
    const size_t per_b = ((bytes + 15) / 16 + m - 1) / m * 16;
    const size_t lo_b = per_b * k < bytes ? per_b * k : bytes;
    const size_t hi_b = lo_b + per_b < bytes ? lo_b + per_b : bytes;
    lo = lo_b / sizeof(U);
    hi = hi_b / sizeof(U);
    for (int j = 1; j < n; ++j) { // other non-roots, starting after me
      const int w = (c.rank + j) % n;
      if (w == root) continue;
      dst[ntargets++] = reinterpret_cast<U*>(c.base[w] + s_a[w]);
    }
  }
  for (int j = ntargets; j < kMaxRanks; ++j) dst[j] = dst[0];
  copy_units<U, UNROLL, kMaxRanks>(src, dst, ntargets, lo, hi);
}

template <typename U, int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
bcast_kernel(Comm c, uint64_t buf_off, size_t bytes, int root, int mode) {
  collective(c, buf_off, buf_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    unit_or_bytes<U, UNROLL>(all_aligned_to(s_a, s_b, c.n, sizeof(U)), [&](auto unit, auto unroll) {
      bcast_body<decltype(unit), unroll>(c, s_a, bytes, root, mode);
    });
  });
}

// Bcast through the switch: root streams its buffer once into the multicast address.
template <int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
bcast_nvls_kernel(Comm c, uint64_t buf_off, size_t bytes, int root) {
  collective(c, buf_off, buf_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    const int n = c.n;
    bool symmetric = (buf_off & 15) == 0 && (bytes & 15) == 0;
    for (int r = 0; r < n; ++r) symmetric = symmetric && s_a[r] == buf_off;
    if (symmetric) {
      if (c.rank == root) {
        const char* src = c.base[root] + buf_off;
        char* dst = c.mc + buf_off;
        unrolled<UNROLL, uint4>(
            0, bytes / 16, [&](size_t i, uint4& v) { v = ldg16(src + i * 16); },
            [&](size_t i, const uint4& v) { multimem_st16(dst + i * 16, v); });
      }
    } else { // different heap offsets per rank: pull from root
      unit_or_bytes<uint4, UNROLL>((bytes & 15) == 0 && all_aligned_to(s_a, s_b, n, 16), [&](auto unit, auto unroll) {
        bcast_body<decltype(unit), unroll>(c, s_a, bytes, root, 0);
      });
    }
  });
}

// Bcast, scatter + multicast: the buffer is cut into ownership blocks (Owner, as in the allreduce);
// the owner of a block fetches it from root with P2P loads (root owns blocks too and reads them
// locally) and multicasts it into every rank's buffer with multimem.st.  Root's link carries every
// byte once (read responses), every other rank's egress is S/n, and all ingress links fill at the
// same time -- the root-only bcast_nvls_kernel is limited by one GPU's multimem.st rate instead.
// Multicast stores also land in root's own buffer: identical bytes over identical bytes.
template <int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
bcast_nvls2_kernel(Comm c, uint64_t buf_off, size_t bytes, int root, uint32_t shift) {
  collective(c, buf_off, buf_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    const int n = c.n;
    bool symmetric = (buf_off & 15) == 0 && (bytes & 15) == 0;
    for (int r = 0; r < n; ++r) symmetric = symmetric && s_a[r] == buf_off;
    if (symmetric) {
      const Owner own(bytes / 16, shift, n, c.rank);
      const char* src = c.base[root] + buf_off;
      char* dst = c.mc + buf_off;
      unrolled_owned<UNROLL, uint4>(
          own, blockIdx.x, gridDim.x, [&](size_t g, uint4& v) { v = ldg16(src + g * 16); }, [&](size_t g, const uint4& v) { multimem_st16(dst + g * 16, v); });
    } else { // different heap offsets per rank: fused P2P two-shot
      unit_or_bytes<uint4, UNROLL>((bytes & 15) == 0 && all_aligned_to(s_a, s_b, n, 16), [&](auto unit, auto unroll) {
        bcast_body<decltype(unit), unroll>(c, s_a, bytes, root, 1);
      });
    }
  });
}

// Allgather through the switch: every rank streams its block once from local HBM into the
// multicast address of its place in the recv buffer; per-GPU egress is one block instead of n-1.
template <int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
allgather_nvls_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t bytes_per_rank) {
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    const int n = c.n;
    bool symmetric = ((recv_off | bytes_per_rank) & 15) == 0;
    for (int r = 0; r < n; ++r) symmetric = symmetric && s_b[r] == recv_off && (s_a[r] & 15) == 0;
    if (symmetric) {
      const char* src = c.base[c.rank] + send_off;
      char* dst = c.mc + recv_off + (size_t)c.rank * bytes_per_rank;
      unrolled<UNROLL, uint4>(
          0, bytes_per_rank / 16, [&](size_t i, uint4& v) { v = ldg16(src + i * 16); }, [&](size_t i, const uint4& v) { multimem_st16(dst + i * 16, v); });
    } else { // different heap offsets per rank: P2P push
      unit_or_bytes<uint4, UNROLL>((bytes_per_rank & 15) == 0 && all_aligned_to(s_a, s_b, n, 16), [&](auto unit, auto unroll) {
        allgather_push_body<decltype(unit), unroll>(c, s_a, s_b, bytes_per_rank);
      });
    }
  });
}

// ---------------------------------------------------------------------------------------------
// Alltoall: block j of rank r's send buffer becomes block r of rank j's recv buffer.  Direct
// push, n write streams per GPU, targets rotated so that the ranks do not all hit one peer.
// ---------------------------------------------------------------------------------------------
// Block j of this rank's send, len(j) bytes at src(j), goes to dst(j) in rank j's heap; targets
// rotated with the own block last (a local copy).  Each block is grid-strided over all CTAs.  The
// loop is written out: through copy_units or `unrolled`, inside this loop over targets, the
// kernels compiled to more registers.
template <typename U, int UNROLL, typename Src, typename Dst, typename Len>
__device__ __forceinline__ void push_rotated(const Comm& c, Src src, Dst dst, Len len) {
  const int n = c.n;
  const size_t step = (size_t)gridDim.x * blockDim.x * UNROLL;
  for (int k = 0; k < n; ++k) {
    const int j = (c.rank + 1 + k) % n; // own block last
    const size_t units = len(j) / sizeof(U);
    const U* s = reinterpret_cast<const U*>(src(j));
    U* d = reinterpret_cast<U*>(dst(j));
    for (size_t i0 = (size_t)blockIdx.x * blockDim.x * UNROLL + threadIdx.x; i0 < units; i0 += step) {
      U v[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < units) v[u] = s[i];
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < units) d[i] = v[u];
      }
    }
  }
}

template <typename U, int UNROLL>
__device__ __forceinline__ void alltoall_body(const Comm& c, const uint64_t* s_a, const uint64_t* s_b, size_t bytes_per_block) {
  push_rotated<U, UNROLL>(
      c, [&](int j) { return c.base[c.rank] + s_a[c.rank] + (size_t)j * bytes_per_block; },
      [&](int j) { return c.base[j] + s_b[j] + (size_t)c.rank * bytes_per_block; }, [&](int) { return bytes_per_block; });
}

template <typename U, int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
alltoall_kernel(Comm c, uint64_t send_off, uint64_t recv_off, size_t bytes_per_block) {
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    unit_or_bytes<U, UNROLL>(all_aligned_to(s_a, s_b, c.n, sizeof(U)), [&](auto unit, auto unroll) {
      alltoall_body<decltype(unit), unroll>(c, s_a, s_b, bytes_per_block);
    });
  });
}

// ---------------------------------------------------------------------------------------------
// Gather(v) / Allgatherv / Scatter(v): blocks of per-rank sizes packed in rank order.  The table is
// the same on every rank (it is part of the call signature), so only the heap offsets can differ.
// ---------------------------------------------------------------------------------------------
struct VTable {
  uint64_t off[kMaxRanks + 1]; // byte displacement of rank r's block; off[n] = total bytes
};

// [off[me], off[me+1]) without indexing the parameter array by a runtime value
__device__ __forceinline__ void vtable_range(const VTable& vt, int me, uint64_t& lo, uint64_t& hi) {
  lo = 0;
  hi = 0;
#pragma unroll
  for (int r = 0; r < kMaxRanks; ++r)
    if (r == me) { lo = vt.off[r]; hi = vt.off[r + 1]; }
}

// Every rank pushes its own block, at its displacement in the table (push_block_body).
template <typename U, int UNROLL>
__device__ __forceinline__ void gatherv_push_body(const Comm& c, const uint64_t* s_a, const uint64_t* s_b, const VTable& vt, int only_dst) {
  uint64_t lo, hi;
  vtable_range(vt, c.rank, lo, hi);
  push_block_body<U, UNROLL>(c, s_a, s_b, lo, hi - lo, only_dst);
}

template <typename U, int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
gatherv_push_kernel(Comm c, uint64_t send_off, uint64_t recv_off, VTable vt, int only_dst) {
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    unit_or_bytes<U, UNROLL>(all_aligned_to(s_a, s_b, c.n, sizeof(U)), [&](auto unit, auto unroll) {
      gatherv_push_body<decltype(unit), unroll>(c, s_a, s_b, vt, only_dst);
    });
  });
}

// Every rank pulls its block [off[rank], off[rank+1]) of root's send through the peer mapping into
// its own recv; root copies its block locally unless the call is in place (recv == send +
// displacement).  Root's egress bounds it either way; pulling spreads the loads over n-1 GPUs.
template <typename U, int UNROLL>
__device__ __forceinline__ void scatterv_pull_body(const Comm& c, const uint64_t* s_a, const uint64_t* s_b, const VTable& vt, int root) {
  uint64_t lo, hi;
  vtable_range(vt, c.rank, lo, hi);
  if (c.rank == root && s_b[root] == s_a[root] + lo) return;
  const size_t units = (hi - lo) / sizeof(U);
  const U* src = reinterpret_cast<const U*>(c.base[root] + s_a[root] + lo);
  U* const dst = reinterpret_cast<U*>(c.base[c.rank] + s_b[c.rank]);
  copy_units<U, UNROLL, 1>(src, &dst, 1, 0, units);
}

template <typename U, int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
scatterv_pull_kernel(Comm c, uint64_t send_off, uint64_t recv_off, VTable vt, int root) {
  collective(c, send_off, recv_off, [&](const uint64_t* s_a, const uint64_t* s_b) {
    unit_or_bytes<U, UNROLL>(all_aligned_to(s_a, s_b, c.n, sizeof(U)), [&](auto unit, auto unroll) {
      scatterv_pull_body<decltype(unit), unroll>(c, s_a, s_b, vt, root);
    });
  });
}

// ---------------------------------------------------------------------------------------------
// ReduceScatterv: rank j receives op over r of block j of rank r's send, combined in rank order,
// where block j is [off[j], off[j+1]) of every send (VTable).  Only rank j reads block j, and each
// element of it is loaded from every rank, reduced and stored by one thread, so recv may be block j
// of rank j's own send (in place) with no mid barrier: the other ranks read only blocks k != j.
// A displacement from a table is rarely a multiple of 16 bytes, so the block is split at the first
// 16-byte boundary of its source addresses (split16): the head and tail elements go one T at a time,
// the whole vectors 16 bytes at a time, as long as the n sources agree mod 16 (heap and staged sends
// are 512-byte aligned and share the displacement, so they usually do).  The vectors are stored 16
// bytes wide when recv has the sources' residue and one T at a time otherwise.  Sources that disagree
// mod 16 leave the whole block to scalar element ownership.
// ---------------------------------------------------------------------------------------------
// `count` elements of `es` bytes from address `addr`: `head` elements up to the first 16-byte
// boundary, `nvec` whole 16-byte vectors from there, `tail` elements after them.  An address that is
// not a multiple of `es` never reaches a boundary on an element edge: everything is head.
struct Split16 {
  size_t head, nvec, tail;
};
__host__ __device__ __forceinline__ Split16 split16(uint64_t addr, size_t count, size_t es) {
  if (addr % es) return {count, 0, 0};
  const size_t head = ((16 - (addr & 15)) & 15) / es;
  if (head >= count) return {count, 0, 0};
  const size_t epv = 16 / es;
  const size_t nvec = (count - head) / epv;
  return {head, nvec, count - head - nvec * epv};
}

// The vector loop loads rank by rank (UNROLL vectors of one rank in flight, then combined), not
// vector by vector as `unrolled` would.  The start/end barriers are written out: through
// `collective` this kernel compiled to different SASS.
template <typename T, typename Op, int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
reduce_scatterv_kernel(Comm c, uint64_t send_off, uint64_t recv_off, VTable vt) {
  __shared__ uint64_t s_a[kMaxRanks], s_b[kMaxRanks];
  __shared__ const char* src[kMaxRanks];
  const bool call_ok = sync_start(c, send_off, recv_off, s_a, s_b);
  if (!call_ok) {
    sync_end_failed(c);
    return;
  }
  const int n = c.n;
  constexpr int EPV = Pack<T>::N;
  uint64_t lo, hi;
  vtable_range(vt, c.rank, lo, hi);
  if (threadIdx.x < (unsigned)n) src[threadIdx.x] = c.base[threadIdx.x] + s_a[threadIdx.x] + lo;
  __syncthreads();
  const size_t count = (hi - lo) / sizeof(T);
  T* const out = reinterpret_cast<T*>(c.base[c.rank] + recv_off);
  const uint64_t res = (send_off + lo) & 15;
  bool agree = true;
  for (int r = 0; r < n; ++r) agree = agree && ((s_a[r] + lo) & 15) == res;
  const Split16 sp = agree ? split16(send_off + lo, count, sizeof(T)) : Split16{count, 0, 0};
  const size_t tid = threadIdx.x;
  const size_t gtid = (size_t)blockIdx.x * blockDim.x + tid, gstride = (size_t)gridDim.x * blockDim.x;
  for (size_t e = gtid; e < sp.head; e += gstride) out[e] = reduce_ranks<T, Op>([&](int r) { return src[r]; }, n, e);
  const size_t v0 = sp.head * sizeof(T); // byte offset of the first whole vector in every source
  const bool wide_out = (recv_off & 15) == res;
  const size_t step = gstride * UNROLL;
  for (size_t i0 = (size_t)blockIdx.x * blockDim.x * UNROLL + tid; i0 < sp.nvec; i0 += step) {
    Pack<T> acc[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t i = i0 + (size_t)u * blockDim.x;
      if (i < sp.nvec) acc[u] = ld_pack<T>(src[0] + v0 + i * 16);
    }
    for (int r = 1; r < n; ++r) { // UNROLL vectors of rank r in flight, combined in rank order
      Pack<T> v[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < sp.nvec) v[u] = ld_pack<T>(src[r] + v0 + i * 16);
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u)
        if (i0 + (size_t)u * blockDim.x < sp.nvec) acc[u] = combine<T, Op>(acc[u], v[u]);
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t i = i0 + (size_t)u * blockDim.x;
      if (i >= sp.nvec) continue;
      if (wide_out) {
        st_pack<T>(reinterpret_cast<char*>(out) + v0 + i * 16, acc[u]);
      } else {
#pragma unroll
        for (int k = 0; k < EPV; ++k) out[sp.head + i * EPV + k] = acc[u].v[k];
      }
    }
  }
  for (size_t e = sp.head + sp.nvec * EPV + gtid; e < count; e += gstride) out[e] = reduce_ranks<T, Op>([&](int r) { return src[r]; }, n, e);
  sync_end(c);
}

// ---------------------------------------------------------------------------------------------
// Alltoallv: rank i holds its send row S_i[0..n) and its recv column R_i[0..n) of an n x n matrix of
// block sizes; the call is consistent when R_j[i] == S_i[j] for every pair.  The tables differ from
// rank to rank, so they cannot be hashed into one shared signature.  Instead rank i announces
// base_sig + D_i with the zero-sum digest
//     D_i = sum_j f(i, j, S_i[j] bytes) - sum_k f(k, i, R_i[k] bytes)   (mod 2^64),
// where every consistent entry appears once with + (at its sender) and once with - (at its
// receiver), so the D_i of a consistent matrix sum to 0 (sync_start_pairs).  For fixed (src, dst),
// f is a bijection of the byte count (xor with a per-pair key, then the splitmix64 finaliser), so a
// change of any single entry always changes the sum; other changes (a swap of two entries) escape
// only by a 64-bit collision, and even then the per-pair byte check keeps every store in bounds.
// ---------------------------------------------------------------------------------------------
__host__ __device__ inline uint64_t a2av_term(int src, int dst, uint64_t bytes) {
  return mix64(bytes ^ mix64(0x616c6c746f616c6cull + (uint64_t)(src * kMaxRanks + dst)));
}

// Rank `me`'s byte displacements (send: of the block for rank j; recv: of the block from rank k; off[n]
// = total, off[r] = total for r > n) and its digest D_me.  false when a count times the element size,
// or a sum of them, does not fit in 64 bits.
__host__ __device__ inline bool a2av_tables(int me, int n, const size_t* send_counts, const size_t* recv_counts, size_t es,
                                            VTable& sv, VTable& rv, uint64_t& digest) {
  uint64_t so = 0, ro = 0, d = 0;
  for (int r = 0; r < n; ++r) {
    sv.off[r] = so;
    rv.off[r] = ro;
    if (send_counts[r] > (UINT64_MAX - so) / es || recv_counts[r] > (UINT64_MAX - ro) / es) return false;
    so += send_counts[r] * es;
    ro += recv_counts[r] * es;
    d += a2av_term(me, r, send_counts[r] * es) - a2av_term(r, me, recv_counts[r] * es);
  }
  for (int r = n; r <= kMaxRanks; ++r) {
    sv.off[r] = so;
    rv.off[r] = ro;
  }
  digest = d;
  return true;
}

// Push: every rank reads its n send blocks once from local HBM and stores block j at s_b[j] of rank
// j's heap (push_rotated), so a skewed table still spreads over the whole grid.  s_src[j] is the
// heap offset of block j in this rank's send, s_len[j] its bytes.
template <typename U, int UNROLL>
__device__ __forceinline__ void alltoallv_push_body(const Comm& c, const uint64_t* s_src, const uint64_t* s_len, const uint64_t* s_b) {
  push_rotated<U, UNROLL>(c, [&](int j) { return c.base[c.rank] + s_src[j]; }, [&](int j) { return c.base[j] + s_b[j]; }, [&](int j) { return s_len[j]; });
}

// sv / rv: this rank's send and recv displacements (a2av_tables); c.sig = base_sig + its digest.
// U was picked by the host from this rank's offsets and displacements; a peer whose destination
// offsets are less aligned sends this rank to the byte-wide body.
template <typename U, int UNROLL>
__global__ void __launch_bounds__(kThreads, 1)
alltoallv_push_kernel(Comm c, uint64_t send_off, uint64_t recv_off, VTable sv, VTable rv, uint64_t base_sig) {
  __shared__ uint64_t s_a[kMaxRanks], s_b[kMaxRanks], s_src[kMaxRanks];
  const int t = threadIdx.x;
  uint64_t slo = 0, shi = 0, rlo = 0, rhi = 0;
  if (t < c.n) {
    vtable_range(sv, t, slo, shi);
    vtable_range(rv, t, rlo, rhi);
    s_src[t] = send_off + slo;
  }
  const bool call_ok = sync_start_pairs(c, base_sig, rhi - rlo, recv_off + rlo, shi - slo, s_a, s_b);
  if (!call_ok) {
    sync_end_failed(c);
    return;
  }
  uint64_t m = 0;
  for (int r = 0; r < c.n; ++r) m |= s_b[r];
  unit_or_bytes<U, UNROLL>((m & (sizeof(U) - 1)) == 0, [&](auto unit, auto unroll) {
    alltoallv_push_body<decltype(unit), unroll>(c, s_src, s_a, s_b);
  });
  sync_end(c);
}

// ---------------------------------------------------------------------------------------------
// Point-to-point and local copies: dst <- src, `bytes` bytes, any alignment.  src may be a peer
// mapping (receiver pulls the sender's posted region over NVLink).
// ---------------------------------------------------------------------------------------------
template <int UNROLL, int THREADS = kThreads, int MINB = 1>
__global__ void __launch_bounds__(THREADS, MINB)
copy_bytes_kernel(unsigned char* __restrict__ dst, const unsigned char* __restrict__ src, size_t bytes) {
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const uintptr_t da = reinterpret_cast<uintptr_t>(dst), sa = reinterpret_cast<uintptr_t>(src);
  if (((da ^ sa) & 15) == 0) {
    size_t head = (16 - (da & 15)) & 15;
    if (head > bytes) head = bytes;
    for (size_t i = tid; i < head; i += stride) dst[i] = src[i];
    const size_t nvec = (bytes - head) / 16;
    const unsigned char* s = src + head;
    unsigned char* d = dst + head;
    unrolled<UNROLL, uint4>(0, nvec, [&](size_t i, uint4& v) { v = ldg16(s + i * 16); }, [&](size_t i, const uint4& v) { stg16(d + i * 16, v); });
    for (size_t i = head + nvec * 16 + tid; i < bytes; i += stride) dst[i] = src[i];
  } else {
    for (size_t i = tid; i < bytes; i += stride) dst[i] = src[i];
  }
}

// ---------------------------------------------------------------------------------------------
// Local copy (both ends in this GPU's memory, (src ^ dst) & 15 == 0): one 16-byte vector per thread
// and a grid that covers the whole message, so the block scheduler hands out CTAs as earlier ones
// retire; there is no grid-stride loop whose last pass runs on a few SMs, and no per-thread burst of
// loads followed by a burst of stores.  Threads 0..15 of CTA 0 also copy the < 16 head and tail
// bytes outside the aligned span.  With a capped grid (b200mpi_set_max_blocks) the loop runs more
// than once.
// ---------------------------------------------------------------------------------------------
constexpr int kLocalCopyThreads = 512;

__global__ void __launch_bounds__(kLocalCopyThreads)
copy_local_kernel(unsigned char* __restrict__ dst, const unsigned char* __restrict__ src, size_t bytes) {
  size_t head = (16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15;
  if (head > bytes) head = bytes;
  const size_t nvec = (bytes - head) / 16;
  const uint4* __restrict__ s = reinterpret_cast<const uint4*>(src + head);
  uint4* __restrict__ d = reinterpret_cast<uint4*>(dst + head);
  const size_t stride = (size_t)gridDim.x * kLocalCopyThreads;
  for (size_t i = (size_t)blockIdx.x * kLocalCopyThreads + threadIdx.x; i < nvec; i += stride) d[i] = s[i];
  if (blockIdx.x == 0 && threadIdx.x < 16) {
    const size_t t = threadIdx.x, tail0 = head + nvec * 16;
    if (t < head) dst[t] = src[t];
    if (tail0 + t < bytes) dst[tail0 + t] = src[tail0 + t];
  }
}

// ---------------------------------------------------------------------------------------------
// Allreduce, LL (low latency): bit-exact against the oracle in worlds of 2 and 4 ranks sharing one
// H100 (tests/test_gpu_worlds.py::test_ll_...); its latency over NVLink has not been measured on
// H100.  AUTO uses it on multi-GPU worlds up to "ll_max_bytes".
// One kernel, no barrier at all.  Every rank pushes its whole (<= 32 KiB) message into a private
// lane of every peer's heap as 16-byte cells {data32, seq, data32, seq} (the NCCL "LL" layout: each
// 8-byte half carries its own flag, so only 8-byte store atomicity is assumed), then reduces its
// own lane set in rank order, spinning per cell until both flags equal this call's sequence number.
// Lanes are double buffered by seq parity: a peer can only be one call ahead, because finishing
// call k+1 needs this rank's k+1 cells, which are sent after this rank finished reading call k.
// Peers never read this rank's send buffer, so there is no end barrier and in place is free; send
// and recv may be any local device pointers.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4* ll_lane(const Comm& c, int owner, uint32_t parity, int src) {
  return reinterpret_cast<uint4*>(c.base[owner] + kLLOff) + ((size_t)parity * c.n + src) * ll_cells(c.n);
}
template <typename T> struct LLCodec; // 8 payload bytes <-> elements
template <> struct LLCodec<float> {
  static constexpr int EPC = 2;
  __device__ __forceinline__ static void pack(const float* e, uint32_t& w0, uint32_t& w1) { w0 = __float_as_uint(e[0]); w1 = __float_as_uint(e[1]); }
  __device__ __forceinline__ static void unpack(uint32_t w0, uint32_t w1, float* e) { e[0] = __uint_as_float(w0); e[1] = __uint_as_float(w1); }
};
template <> struct LLCodec<double> {
  static constexpr int EPC = 1;
  __device__ __forceinline__ static void pack(const double* e, uint32_t& w0, uint32_t& w1) { unsigned long long b = (unsigned long long)__double_as_longlong(e[0]); w0 = (uint32_t)b; w1 = (uint32_t)(b >> 32); }
  __device__ __forceinline__ static void unpack(uint32_t w0, uint32_t w1, double* e) { e[0] = __longlong_as_double((long long)(((unsigned long long)w1 << 32) | w0)); }
};
template <> struct LLCodec<long long> {
  static constexpr int EPC = 1;
  __device__ __forceinline__ static void pack(const long long* e, uint32_t& w0, uint32_t& w1) { unsigned long long b = (unsigned long long)e[0]; w0 = (uint32_t)b; w1 = (uint32_t)(b >> 32); }
  __device__ __forceinline__ static void unpack(uint32_t w0, uint32_t w1, long long* e) { e[0] = (long long)(((unsigned long long)w1 << 32) | w0); }
};

template <typename T, typename Op>
__global__ void __launch_bounds__(256, 1)
allreduce_ll_kernel(Comm c, const T* __restrict__ send, T* recv, size_t count, uint32_t seq, uint32_t* done_host) {
  constexpr int EPC = LLCodec<T>::EPC;
  const size_t ncell = (count + EPC - 1) / EPC;
  const uint32_t parity = seq & 1u;
  const int n = c.n;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  // phase 1: every cell of this thread goes out to every peer before anything is waited for, so a
  // message of many cells costs one exchange latency, not one per cell
  for (size_t i = tid; i < ncell; i += stride) {
    T mine[EPC];
#pragma unroll
    for (int k = 0; k < EPC; ++k) mine[k] = i * EPC + k < count ? send[i * EPC + k] : T(0);
    uint32_t w0, w1;
    LLCodec<T>::pack(mine, w0, w1);
    const uint4 cell = make_uint4(w0, seq, w1, seq);
    for (int j = 1; j < n; ++j) { // push to every peer, starting after this rank
      const int r = (c.rank + j) % n;
      st_cell16(ll_lane(c, r, parity, c.rank) + i, cell);
    }
  }
  // phase 2: reduce the own lanes in rank order.  The n-1 cells of one element are loaded together
  // (independent loads in flight: one L2 latency, not n-1) and re-loaded only while their flags lag.
  for (size_t i = tid; i < ncell; i += stride) {
    T mine[EPC];
#pragma unroll
    for (int k = 0; k < EPC; ++k) mine[k] = i * EPC + k < count ? send[i * EPC + k] : T(0);
    uint4 got[kMaxRanks];
    uint32_t pending = 0;
#pragma unroll
    for (int r = 0; r < kMaxRanks; ++r)
      if (r < n && r != c.rank) {
        got[r] = ld_cell16(ll_lane(c, c.rank, parity, r) + i);
        pending |= 1u << r;
      }
    // the watchdog poll of wait_flag
    unsigned long long t0 = 0;
    uint32_t it = 0;
    for (;;) {
#pragma unroll
      for (int r = 0; r < kMaxRanks; ++r)
        if ((pending >> r) & 1u) {
          if (got[r].y == seq && got[r].w == seq) pending &= ~(1u << r);
        }
      if (!pending) break;
#pragma unroll
      for (int r = 0; r < kMaxRanks; ++r)
        if ((pending >> r) & 1u) got[r] = ld_cell16(ll_lane(c, c.rank, parity, r) + i);
      if ((++it & 0xfffu) == 0) {
        const unsigned long long now = globaltimer_ns();
        if (t0 == 0) t0 = now;
        else if (c.timeout_ns && now - t0 > c.timeout_ns) {
          *(volatile uint32_t*)c.status = 1u;
          __threadfence_system();
          break;
        }
      }
    }
    T acc[EPC];
#pragma unroll
    for (int r = 0; r < kMaxRanks; ++r)
      if (r < n) {
        T v[EPC];
        if (r == c.rank) {
#pragma unroll
          for (int k = 0; k < EPC; ++k) v[k] = mine[k];
        } else {
          LLCodec<T>::unpack(got[r].x, got[r].z, v);
        }
#pragma unroll
        for (int k = 0; k < EPC; ++k) acc[k] = r == 0 ? v[k] : Op::template apply<T>(acc[k], v[k]);
      }
#pragma unroll
    for (int k = 0; k < EPC; ++k)
      if (i * EPC + k < count) recv[i * EPC + k] = acc[k];
  }
  // Host-slice calls: send/recv are device-mapped pinned host buffers and the caller spins on
  // *done_host instead of paying a stream synchronisation.  The last CTA to finish publishes seq
  // after every CTA's result stores have been fenced at system scope.
  if (done_host) {
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned* ctas = reinterpret_cast<unsigned*>(c.base[c.rank] + kLLStateOff);
      __threadfence_system();
      if (atomicAdd(ctas, 1u) == gridDim.x - 1) {
        *ctas = 0;
        __threadfence_system();
        *(volatile uint32_t*)done_host = seq;
      }
    }
  }
}

// Completion word for host-polled copies: enqueued right behind a copy kernel on the same stream, so
// the copy's stores (possibly into mapped host memory) are complete when the word becomes visible.
__global__ void flag_kernel(uint32_t* done, uint32_t value) {
  __threadfence_system();
  *(volatile uint32_t*)done = value;
}

// Flag words are compared wrap-safe ((int32_t)(flag - want) >= 0), which is only sound while no word lags
// the epoch by 2^31.  A slot row of a block index that has not been used for 2^31 / kEpochStride =
// 524,288 launches would look "ahead" (65,536 for the ring step counters, which count epoch * 8).
// Every kScrubEvery launches the host therefore runs this
// kernel with the largest grid: its start and end barriers rewrite the cells and the flag of every
// row on every rank, and each CTA refreshes its ring step counter.
__global__ void scrub_kernel(Comm c) {
  __shared__ uint64_t s_a[kMaxRanks], s_b[kMaxRanks];
  const bool ok = sync_start(c, 0, 0, s_a, s_b);
  if (threadIdx.x == 0) *ring_flag(c, c.rank, blockIdx.x) = c.epoch * 8u;
  if (ok) sync_end(c);
  else sync_end_failed(c);
}

// A device-wide rendezvous with nothing in between (b200mpi_barrier, and b200mpi_win_fence under its
// own signature).
__global__ void barrier_kernel(Comm c) {
  collective(c, 0, 0, [](const uint64_t*, const uint64_t*) {});
}

// ---------------------------------------------------------------------------------------------
// One-sided Accumulate (b200mpi_accumulate): dst[e] = Op(dst[e], src[e]) for every element, each an
// atomic read-modify-write at system scope, where dst is the target's window through its peer
// mapping and src this rank's origin (or its staging block) in local HBM.  Concurrent Accumulates with
// the same type and op from any ranks therefore combine in some order, none lost.
//   sums and i64 max/min: fire-and-forget `red`.  f32 sum has a 16-byte form; sm_90a flushes f32
//     atomic add inputs and results that are subnormal to zero of the same sign (there is no .noftz
//     f32 red), so an f32 Accumulate SUM differs there from Allreduce, which keeps subnormals.
//   replace (B200MPI_REPLACE): an element-wise st.relaxed.sys.
//   f32 / f64 max and min: an atom.cas loop that applies OpMax / OpMin (b > a ? b : a), so a NaN
//     already in the target stays and a NaN contribution is dropped; the result depends on the order
//     of contributions only through NaNs and zeros of mixed sign.
// ---------------------------------------------------------------------------------------------
template <typename T, typename Op>
struct Red { // f32 / f64 max and min
  using Bits = std::conditional_t<sizeof(T) == 4, uint32_t, unsigned long long>;
  __device__ __forceinline__ static void one(T* p, T v) { (void)fetch(p, v); }
  // The CAS loop; returns the value its successful compare-and-swap saw (Get_accumulate's result).
  __device__ __forceinline__ static T fetch(T* p, T v) {
    Bits old;
    if constexpr (sizeof(T) == 4) asm volatile("ld.relaxed.sys.global.b32 %0, [%1];" : "=r"(old) : "l"(p) : "memory");
    else asm volatile("ld.relaxed.sys.global.b64 %0, [%1];" : "=l"(old) : "l"(p) : "memory");
    for (;;) {
      T cur, next;
      memcpy(&cur, &old, sizeof(T));
      next = Op::template apply<T>(cur, v);
      Bits want, seen;
      memcpy(&want, &next, sizeof(T));
      // No early exit when want == old: only a successful compare-and-swap proves that `old` was the
      // target's value, so the result never rests on the load above being current.
      if constexpr (sizeof(T) == 4)
        asm volatile("atom.relaxed.sys.global.cas.b32 %0, [%1], %2, %3;" : "=r"(seen) : "l"(p), "r"(old), "r"(want) : "memory");
      else
        asm volatile("atom.relaxed.sys.global.cas.b64 %0, [%1], %2, %3;" : "=l"(seen) : "l"(p), "l"(old), "l"(want) : "memory");
      if (seen == old) return cur;
      old = seen;
    }
  }
};
template <> struct Red<float, OpSum> {
  __device__ __forceinline__ static void one(float* p, float v) {
    asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
  }
  __device__ __forceinline__ static void vec(float* p, const Pack<float>& v) {
    asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.v[0]), "f"(v.v[1]), "f"(v.v[2]), "f"(v.v[3]) : "memory");
  }
};
template <> struct Red<double, OpSum> {
  __device__ __forceinline__ static void one(double* p, double v) {
    asm volatile("red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
  }
};
template <> struct Red<long long, OpSum> { // wraps, as Go int64 does
  __device__ __forceinline__ static void one(long long* p, long long v) {
    asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
  }
};
template <> struct Red<long long, OpMax> {
  __device__ __forceinline__ static void one(long long* p, long long v) {
    asm volatile("red.relaxed.sys.global.max.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
  }
};
template <> struct Red<long long, OpMin> {
  __device__ __forceinline__ static void one(long long* p, long long v) {
    asm volatile("red.relaxed.sys.global.min.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
  }
};

template <typename T> struct Red<T, OpReplace> { // MPI_REPLACE: an element-wise atomic store
  __device__ __forceinline__ static void one(T* p, T v) {
    if constexpr (sizeof(T) == 4) {
      uint32_t b;
      memcpy(&b, &v, 4);
      asm volatile("st.relaxed.sys.global.b32 [%0], %1;" ::"l"(p), "r"(b) : "memory");
    } else {
      unsigned long long b;
      memcpy(&b, &v, 8);
      asm volatile("st.relaxed.sys.global.b64 [%0], %1;" ::"l"(p), "l"(b) : "memory");
    }
  }
};

// One 16-byte vector: the 16-byte red where there is one (f32 sum), else one element at a time.
template <typename T, typename Op>
__device__ __forceinline__ void red_vec(T* p, const Pack<T>& v) {
  if constexpr (std::is_same<T, float>::value && std::is_same<Op, OpSum>::value) {
    Red<T, Op>::vec(p, v);
  } else {
#pragma unroll
    for (int k = 0; k < Pack<T>::N; ++k) Red<T, Op>::one(p + k, v.v[k]);
  }
}

// `count` elements; dst is element aligned (checked by the host), src element aligned too (a heap
// origin that is not is staged first).  The target is split at its first 16-byte boundary (split16):
// head and tail elements one at a time, the whole vectors between them 16 bytes at a time when src
// has dst's residue mod 16, otherwise every element one at a time.  Grid-strided: a capped grid
// (b200mpi_set_max_blocks) makes several passes.
template <typename T, typename Op>
__global__ void __launch_bounds__(256, 1)
accumulate_kernel(T* dst, const T* __restrict__ src, size_t count) {
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  constexpr int EPV = Pack<T>::N;
  const bool agree = ((reinterpret_cast<uintptr_t>(dst) ^ reinterpret_cast<uintptr_t>(src)) & 15) == 0;
  const Split16 sp = agree ? split16(reinterpret_cast<uintptr_t>(dst), count, sizeof(T)) : Split16{count, 0, 0};
  for (size_t e = tid; e < sp.head; e += stride) Red<T, Op>::one(dst + e, src[e]);
  T* const d = dst + sp.head;
  const T* const s = src + sp.head;
  unrolled<4, Pack<T>>(0, sp.nvec, [&](size_t i, Pack<T>& v) { v = ld_pack<T>(s + i * EPV); },
                       [&](size_t i, const Pack<T>& v) { red_vec<T, Op>(d + i * EPV, v); });
  for (size_t e = sp.head + sp.nvec * EPV + tid; e < count; e += stride) Red<T, Op>::one(dst + e, src[e]);
}

// ---------------------------------------------------------------------------------------------
// Passive target (b200mpi_get_accumulate, _fetch_and_op, _compare_and_swap, _win_lock / _unlock).
// Fetch<T, Op>::one(p, v) is one fetching atomic at system scope that applies Op and returns the
// element's previous bits: atom.add (f32, f64, u64), atom.max / min.s64, Red's CAS loop for float max
// and min, atom.exch for REPLACE, an ld.relaxed.sys for NO_OP.  The same instruction at the same
// address and width as Accumulate's red, so the two are atomic with respect to each other.  atom.add.f32
// flushes subnormal inputs and results, as red does; the value it returns is the old bits as stored.
// ---------------------------------------------------------------------------------------------
template <typename T, typename Op>
struct Fetch { // f32 / f64 max and min
  __device__ __forceinline__ static T one(T* p, T v) { return Red<T, Op>::fetch(p, v); }
};
template <> struct Fetch<float, OpSum> {
  __device__ __forceinline__ static float one(float* p, float v) {
    float old;
    asm volatile("atom.relaxed.sys.global.add.f32 %0, [%1], %2;" : "=f"(old) : "l"(p), "f"(v) : "memory");
    return old;
  }
};
template <> struct Fetch<double, OpSum> {
  __device__ __forceinline__ static double one(double* p, double v) {
    double old;
    asm volatile("atom.relaxed.sys.global.add.f64 %0, [%1], %2;" : "=d"(old) : "l"(p), "d"(v) : "memory");
    return old;
  }
};
template <> struct Fetch<long long, OpSum> { // wraps
  __device__ __forceinline__ static long long one(long long* p, long long v) {
    long long old;
    asm volatile("atom.relaxed.sys.global.add.u64 %0, [%1], %2;" : "=l"(old) : "l"(p), "l"(v) : "memory");
    return old;
  }
};
template <> struct Fetch<long long, OpMax> {
  __device__ __forceinline__ static long long one(long long* p, long long v) {
    long long old;
    asm volatile("atom.relaxed.sys.global.max.s64 %0, [%1], %2;" : "=l"(old) : "l"(p), "l"(v) : "memory");
    return old;
  }
};
template <> struct Fetch<long long, OpMin> {
  __device__ __forceinline__ static long long one(long long* p, long long v) {
    long long old;
    asm volatile("atom.relaxed.sys.global.min.s64 %0, [%1], %2;" : "=l"(old) : "l"(p), "l"(v) : "memory");
    return old;
  }
};
template <typename T> struct Fetch<T, OpReplace> {
  __device__ __forceinline__ static T one(T* p, T v) {
    T r;
    if constexpr (sizeof(T) == 4) {
      uint32_t b, old;
      memcpy(&b, &v, 4);
      asm volatile("atom.relaxed.sys.global.exch.b32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(b) : "memory");
      memcpy(&r, &old, 4);
    } else {
      unsigned long long b, old;
      memcpy(&b, &v, 8);
      asm volatile("atom.relaxed.sys.global.exch.b64 %0, [%1], %2;" : "=l"(old) : "l"(p), "l"(b) : "memory");
      memcpy(&r, &old, 8);
    }
    return r;
  }
};
template <typename T> struct Fetch<T, OpNoOp> { // an atomic read
  __device__ __forceinline__ static T one(T* p, T) {
    T r;
    if constexpr (sizeof(T) == 4) {
      uint32_t old;
      asm volatile("ld.relaxed.sys.global.b32 %0, [%1];" : "=r"(old) : "l"(p) : "memory");
      memcpy(&r, &old, 4);
    } else {
      unsigned long long old;
      asm volatile("ld.relaxed.sys.global.b64 %0, [%1];" : "=l"(old) : "l"(p) : "memory");
      memcpy(&r, &old, 8);
    }
    return r;
  }
};

// res[e] = dst[e] before, dst[e] = Op(dst[e], src[e]), one element per thread, grid-strided over
// copy_grid.  dst (the target through its peer mapping), src and res are element aligned (the host
// stages misaligned heap buffers); res == src is in place (each thread reads its src element before
// it writes that res element); src is not read for NO_OP and may be null then.  No vector form:
// these calls are latency-bound.
template <typename T, typename Op>
__global__ void __launch_bounds__(256, 1)
get_accumulate_kernel(T* dst, const T* src, T* res, size_t count) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < count; e += stride) {
    T v{};
    if constexpr (!std::is_same<Op, OpNoOp>::value) v = src[e];
    res[e] = Fetch<T, Op>::one(dst + e, v);
  }
}

// One element, the operand as a parameter and the old value to *out, a host-mapped word
// (b200mpi_fetch_and_op: one launch, no staging).  One thread.
template <typename T, typename Op>
__global__ void fetch_op_kernel(T* dst, T v, T* out) {
  *(volatile T*)out = Fetch<T, Op>::one(dst, v);
}

// b200mpi_compare_and_swap: *out = old; dst = v if old == cmp.  One thread, i64 only.
__global__ void cas_kernel(unsigned long long* dst, unsigned long long cmp, unsigned long long v, unsigned long long* out) {
  unsigned long long old;
  asm volatile("atom.relaxed.sys.global.cas.b64 %0, [%1], %2, %3;" : "=l"(old) : "l"(dst), "l"(cmp), "l"(v) : "memory");
  *(volatile unsigned long long*)out = old;
}

// Window locks: one 64-bit word per live window in every rank's control region, past the LL cells.
// Bit 32 is the exclusive holder, the low 32 bits count shared holders (and shared attempts in
// passing, which back out when they find the exclusive bit).
//   exclusive acquire: atom.cas.acquire.sys from 0;      release: atom.and.release.sys of ~bit 32
//     (only its own bit: a shared attempt may have incremented the count in passing)
//   shared acquire: atom.add.acquire.sys of +1, backed out and retried if the exclusive bit was set;
//     release: atom.add.release.sys of -1
constexpr size_t kWinLockOff = 9u << 20;
constexpr size_t kWinLockStride = 64;
constexpr uint32_t kWinLockCells = 65536; // windows live at once; the table ends at 13 MiB
constexpr unsigned long long kLockExclusive = 1ull << 32;
static_assert(kWinLockOff >= kLLOff + kLLRegionCells * 16, "lock words overlap the LL cells");
static_assert(kWinLockOff + (size_t)kWinLockCells * kWinLockStride <= kCtrlBytes, "lock words end past the control region");
// Attempts one win_lock_try_kernel makes, with __nanosleep backoff from 32 ns doubling to 1 us (about
// 0.25 ms in all), before it reports "not acquired" and the host relaunches it.  A guess, not a
// measurement: it bounds the kernel, and the host's deadline (watchdog_ms) bounds the wait.
constexpr int kLockAttempts = 256;

// One thread: up to kLockAttempts tries at the lock word, then *acquired (host-mapped) = 1 or 0.  It
// never spins without bound, and neither touches the device watchdog nor its status word: a rank
// waiting on a lock is not a collective that failed.
__global__ void win_lock_try_kernel(unsigned long long* word, int exclusive, uint32_t* acquired) {
  unsigned ns = 32;
  for (int i = 0; i < kLockAttempts; ++i) {
    unsigned long long old;
    if (exclusive) {
      asm volatile("atom.acquire.sys.global.cas.b64 %0, [%1], %2, %3;" : "=l"(old) : "l"(word), "l"(0ull), "l"(kLockExclusive) : "memory");
      if (old == 0) { *(volatile uint32_t*)acquired = 1; return; }
    } else {
      asm volatile("atom.acquire.sys.global.add.u64 %0, [%1], %2;" : "=l"(old) : "l"(word), "l"(1ull) : "memory");
      if (!(old & kLockExclusive)) { *(volatile uint32_t*)acquired = 1; return; }
      asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(word), "l"(~0ull) : "memory");
    }
    __nanosleep(ns);
    if (ns < 1024) ns *= 2;
  }
  *(volatile uint32_t*)acquired = 0;
}

// One thread: releases what win_lock_try_kernel acquired.  The release orders this rank's earlier RMA
// kernels before the next holder's acquire: they completed before this kernel started (DESIGN §3).
__global__ void win_unlock_kernel(unsigned long long* word, int exclusive) {
  unsigned long long old;
  if (exclusive) asm volatile("atom.release.sys.global.and.b64 %0, [%1], %2;" : "=l"(old) : "l"(word), "l"(~kLockExclusive) : "memory");
  else asm volatile("atom.release.sys.global.add.u64 %0, [%1], %2;" : "=l"(old) : "l"(word), "l"(~0ull) : "memory");
}

// ---------------------------------------------------------------------------------------------
// Generalized active target (b200mpi_win_post / _start / _complete / _wait / _test).  Two 16-bit
// counters per pair of ranks and window, in the window's lock cell past the lock word:
//   posted[t]    in origin o's cell, written only by target t: the exposure epochs t opened to o
//   completed[o] in target t's cell, written only by origin o: the access epochs o closed on t
// Each writer stores a count the host already knows, so no read-modify-write is needed.  A counter
// never runs more than one ahead of its reader's expectation (DESIGN §3), so a poll tests for
// equality with that count, modulo 2^16.
// ---------------------------------------------------------------------------------------------
constexpr size_t kPscwPostedOff = 8;     // u16 posted[kMaxRanks]
constexpr size_t kPscwCompletedOff = 24; // u16 completed[kMaxRanks]
static_assert(kPscwPostedOff >= sizeof(unsigned long long), "PSCW counters overlap the lock word");
static_assert(kPscwCompletedOff >= kPscwPostedOff + kMaxRanks * sizeof(uint16_t), "posted and completed counters overlap");
static_assert(kPscwCompletedOff + kMaxRanks * sizeof(uint16_t) <= kWinLockStride, "PSCW counters end past the window's cell");
// Attempts one pscw_poll_kernel makes at each word, with the lock's __nanosleep backoff (about 0.25
// ms in all), before it reports the members still missing and the host relaunches it.  A guess, not
// a measurement, as kLockAttempts is: it bounds the kernel, and watchdog_ms bounds the wait.
constexpr int kPscwAttempts = 256;

// One entry per group member: the counter word (a peer's cell for a signal, this rank's own cell for
// a poll) and the count to store or to wait for.
struct PscwGroup {
  uint16_t* word[kMaxRanks];
  uint16_t count[kMaxRanks];
};

// Post and complete, one thread per member: st.release.sys of the new count.  The release orders this
// rank's earlier window work before the peer's acquire: those kernels completed before this one
// started, as for win_unlock_kernel.
__global__ void pscw_signal_kernel(const __grid_constant__ PscwGroup grp) {
  const int i = threadIdx.x;
  asm volatile("st.release.sys.global.u16 [%0], %1;" ::"l"(grp.word[i]), "h"(grp.count[i]) : "memory");
}

// Start, wait and test, one thread per member: up to `attempts` ld.acquire.sys of its word, then
// arrived[i] (host-mapped) = 1 if the word held its count, else 0.  Bounded, and it touches neither
// the device watchdog nor the status word: a rank waiting for its peers is not a collective that
// failed.
__global__ void pscw_poll_kernel(const __grid_constant__ PscwGroup grp, int attempts, uint8_t* arrived) {
  const int i = threadIdx.x;
  unsigned ns = 32;
  for (int a = 0; a < attempts; ++a) {
    uint16_t v;
    asm volatile("ld.acquire.sys.global.u16 %0, [%1];" : "=h"(v) : "l"(grp.word[i]) : "memory");
    if (v == grp.count[i]) { *(volatile uint8_t*)(arrived + i) = 1; return; }
    if (a + 1 < attempts) __nanosleep(ns);
    if (ns < 1024) ns *= 2;
  }
  *(volatile uint8_t*)(arrived + i) = 0;
}

} // namespace b200
