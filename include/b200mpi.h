/*
 * b200mpi.h -- C ABI of libb200mpi.so: the H100-native transport that sits behind the
 * btracey/mpi Go facade (mpi.Init/Finalize/Rank/Size/Send/Receive + the new
 * Recv/Bcast/Allreduce/Allgather entry points).
 *
 * This is the drop-in boundary.  Every entry point is what the cgo shim (go/mpi/cuda.go,
 * see INTEGRATION.md) binds for one method of the reference's `mpi.Interface`
 * (/root/reference/mpi.go:163-170) or for one of the collectives the reference only stubs
 * (/root/reference/mpi.go:130, mpi.go:69-71).  Plain pointers and sizes only; no C++ or torch
 * types cross this line.
 *
 * Conventions
 *   - every call returns 0 (B200MPI_OK) or a negative b200mpi_error; the text of the last
 *     error on the calling thread is b200mpi_last_error().
 *   - all data calls block until the caller's buffers may be reused (mpi.go:47-48), except the
 *     *_async forms which only enqueue on the library stream (b200mpi_stream_sync completes them).
 *   - caller owns every buffer; HOST pointers are used only for the duration of the call
 *     (cgo pointer-passing rule); count==0 with buf==NULL is legal (bounce.go:33 sends length 0).
 *   - p2p calls (send/recv) are thread-safe provided {peer,tag} pairs are unique among
 *     in-flight calls (mpi.go:121-125); collectives are called by one thread per rank, in the
 *     same order on every rank.
 */
#ifndef B200MPI_H_
#define B200MPI_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200MPI_VERSION 200 /* 0.2.0: + isend/wait, reduce_scatter, reduce, alltoall, probes, get_param;
                               then gather, scatter, gatherv, scatterv, allgatherv, alltoallv, scan, exscan,
                               reduce_scatterv, allreduce_loc, reduce_loc, win_create, win_free, win_fence,
                               put, get, accumulate, win_lock, win_unlock, get_accumulate, fetch_and_op,
                               compare_and_swap, win_post, win_start, win_complete, win_wait, win_test
                               (all additive) */
#define B200MPI_MAX_RANKS 8 /* "the 8 GPUs of one box" */

typedef enum {
  B200MPI_U8 = 0,  /* []byte / mpi.Raw / gob-encoded anything-else (e.g. string) */
  B200MPI_I64 = 1, /* []int64   */
  B200MPI_F32 = 2, /* []float32 */
  B200MPI_F64 = 3  /* []float64 */
} b200mpi_dtype;

typedef enum { B200MPI_SUM = 0, B200MPI_MAX = 1, B200MPI_MIN = 2,
               B200MPI_REPLACE = 3, /* one-sided only: target = origin */
               B200MPI_NO_OP = 4    /* get_accumulate / fetch_and_op only: target unchanged (atomic read) */
} b200mpi_op; /* every collective takes SUM, MAX and MIN only: REPLACE and NO_OP are B200MPI_ERR_ARG there */
typedef enum { B200MPI_LOCK_EXCLUSIVE = 1, B200MPI_LOCK_SHARED = 2 } b200mpi_lock_type;

typedef enum {
  B200MPI_HOST = 0,  /* pageable or pinned host memory (a Go slice) */
  B200MPI_DEVICE = 1 /* device memory; zero-copy when it lies inside the b200mpi_alloc heap */
} b200mpi_memkind;

typedef enum {
  B200MPI_COLL_ALLREDUCE = 0,
  B200MPI_COLL_BCAST = 1,
  B200MPI_COLL_ALLGATHER = 2,
  B200MPI_COLL_REDUCE_SCATTER = 3
} b200mpi_coll;

typedef enum {
  B200MPI_ALGO_AUTO = 0,    /* size/topology based choice (default) */
  B200MPI_ALGO_ONESHOT = 1, /* allreduce: every rank reads all n buffers (latency path);
                               bcast: everyone pulls from root; allgather: direct push */
  B200MPI_ALGO_TWOSHOT = 2, /* allreduce: owner-reduces-slice + push to all, one fused pass;
                               bcast: pull-slice-from-root + push to all, one fused pass */
  B200MPI_ALGO_RING = 3,    /* allreduce/allgather: 2(n-1) / (n-1) neighbour steps */
  B200MPI_ALGO_NVLS = 4,    /* multimem.ld_reduce / multimem.st through the NVSwitch */
  B200MPI_ALGO_TWOSHOT_SMEM = 5, /* allreduce two-shot with cp.async.bulk shared-memory staging */
  B200MPI_ALGO_LL = 6,       /* allreduce <= 256 KiB: flag-in-data cells, no barrier (the small-message default) */
  B200MPI_ALGO_HYBRID = 7    /* allreduce: NVLS for most of the message + fused P2P two-shot for the rest, one kernel */
} b200mpi_algo;

typedef enum {
  B200MPI_OK = 0,
  B200MPI_ERR_ARG = -1,         /* bad argument (rank/dtype/op/NULL with count>0 ...) */
  B200MPI_ERR_NOT_INIT = -2,    /* call before init / after finalize */
  B200MPI_ERR_BOOTSTRAP = -3,   /* address list / listen / dial / handshake failure */
  B200MPI_ERR_PASSWORD = -4,    /* "bad password" (network.go:343-346) */
  B200MPI_ERR_TIMEOUT = -5,     /* init timeout (network.go:223-231) or device-flag watchdog */
  B200MPI_ERR_TAG_EXISTS = -6,  /* duplicate in-flight {peer,tag} (mpi.go:174-182) */
  B200MPI_ERR_CUDA = -7,        /* a CUDA runtime/driver call failed */
  B200MPI_ERR_NOMEM = -8,       /* symmetric heap exhausted */
  B200MPI_ERR_TRUNCATE = -9,    /* recv capacity smaller than the message */
  B200MPI_ERR_NO_DEVICE = -10,  /* no usable CUDA device (there is no CPU fallback) */
  B200MPI_ERR_UNSUPPORTED = -11,/* dtype/op/algo combination not implemented */
  B200MPI_ERR_PEER = -12        /* a peer reported failure / mismatched collective */
} b200mpi_error;

/* ---- lifecycle: mpi.Init / Finalize / Rank / Size  (mpi.go:96-118, network.go:41-65) -------- */

/* addr / alladdr_csv / password / timeout_ns are the values of -mpi-addr, -mpi-alladdr,
 * -mpi-password, -mpi-inittimeout (flags.go:44-50).  Empty alladdr_csv => single rank on
 * ":5000" (network.go:55-58).  rank = index of addr in the sorted address list
 * (network.go:94-109).  gpu: device ordinal, -1 = rank % deviceCount.
 * gpu == -2 starts the control plane only (no CUDA): rank/size/barrier work, data calls
 * return B200MPI_ERR_NO_DEVICE.  Used by CPU-only plumbing tests. */
int b200mpi_init(const char* addr, const char* alladdr_csv, const char* password,
                 int64_t timeout_ns, int gpu);
int b200mpi_finalize(void);
int b200mpi_rank(void); /* -1 before init (mpi.go:110-112) */
int b200mpi_size(void); /*  0 before init (mpi.go:116-118) */
int b200mpi_device(void); /* CUDA ordinal bound to this rank, -1 if none */
int b200mpi_version(void);
const char* b200mpi_last_error(void); /* thread-local, never NULL */

/* ---- memory -------------------------------------------------------------------------------- */

/* Device memory from this rank's peer-mapped heap (size: env B200MPI_HEAP_BYTES, default 2 GiB).
 * Buffers from here take the zero-copy path; any other device pointer is staged through it. */
int b200mpi_alloc(size_t bytes, void** dptr);
int b200mpi_free(void* dptr);
/* Pinned host memory on the NUMA node of this rank's GPU (optional; plain malloc'ed / Go memory
 * works too: it is staged through a pinned bounce ring by helper threads). */
int b200mpi_host_alloc(size_t bytes, void** hptr);
int b200mpi_host_free(void* hptr);
/* Synchronous copies for harnesses that have no CUDA binding of their own. kind: 0 H2D, 1 D2H, 2 D2D */
int b200mpi_memcpy(void* dst, const void* src, size_t bytes, int kind);
int b200mpi_heap_info(size_t* total, size_t* used, int* nvls_available);
int b200mpi_numa_node(void); /* NUMA node of the bound GPU (sysfs), -1 unknown */

/* ---- point to point: mpi.Send / mpi.Receive (mpi.go:126,157; network.go:518-602) ----------- */

/* Synchronous (rendezvous) send: returns once the matching recv has taken the data, like the
 * reference's ack wait (network.go:569).  dest == own rank is legal (network.go:545-548). */
int b200mpi_send(const void* buf, size_t count, int dtype, int dest, int tag, int memkind);
/* The Send/Wait pair sketched in the reference (mpi.go:132-152, commented out there): isend
 * returns once the data has left the caller's buffer ("sent on connection", here: staged in this
 * rank's device heap), without waiting for the receiver; wait blocks until `dest` confirmed the
 * message with `tag` and frees the {dest, tag} pair.  Every isend must be followed by one wait.
 * Each (rank, dest) pair has 16 mailbox slots; a send holds one until it returns, an isend until its
 * wait, whether or not the message was received.  So at most 16 isends to one dest may be unwaited:
 * the 17th finds no free slot and fails with B200MPI_ERR_TIMEOUT after the watchdog time. */
int b200mpi_isend(const void* buf, size_t count, int dtype, int dest, int tag, int memkind);
int b200mpi_wait(int dest, int tag);
/* Blocks for message (src, tag).  *count_out = elements sent (gob resizes the destination,
 * network.go:597); more than `capacity` elements => B200MPI_ERR_TRUNCATE, *count_out = needed.
 * A host buffer is filled through a staging block of at most "stage_chunk" bytes (32 MiB) in this
 * rank's heap, whatever memory the sender passed; without room for it => B200MPI_ERR_NOMEM.  After
 * either error nothing is written and the message stays posted: receive it again. */
int b200mpi_recv(void* buf, size_t capacity, size_t* count_out, int dtype, int src, int tag,
                 int memkind);

/* ---- collectives (new API; semantics in SURVEY.md 8(c), oracle/collectives.c) -------------- */

/* Bcast, Allreduce and Allgather of host memory from "pipe_min_bytes" (8 MiB, the whole recv for
 * Allgather) up run a chunked pipeline: one launch per chunk, where device memory runs one launch.  There
 * every rank must pass the same memkind.  Pageable, pinned and registered host memory may be mixed
 * across ranks: in a multi-rank world all of them use the same chunks. */
int b200mpi_bcast(void* buf, size_t count, int dtype, int root, int memkind);
/* send == recv means in place. */
int b200mpi_allreduce(const void* send, void* recv, size_t count, int dtype, int op, int memkind);
/* recv holds size()*count_per_rank elements, rank r's block at r*count_per_rank. */
int b200mpi_allgather(const void* send, void* recv, size_t count_per_rank, int dtype, int memkind);
/* send holds size()*count_per_rank elements; rank j receives op over r of rank r's block j
 * (rank order).  recv may be the caller's own block of send (in place).  This is the first half
 * of the two-shot Allreduce on its own. */
int b200mpi_reduce_scatter(const void* send, void* recv, size_t count_per_rank, int dtype, int op, int memkind);
/* Allreduce whose result lands on `root` only (recv may be NULL elsewhere). */
int b200mpi_reduce(const void* send, void* recv, size_t count, int dtype, int op, int root, int memkind);
/* send and recv hold size()*count_per_rank elements; block j of send becomes block rank() of rank j's recv. */
int b200mpi_alltoall(const void* send, void* recv, size_t count_per_rank, int dtype, int memkind);
/* recv (root only, may be NULL elsewhere) holds size()*count_per_rank; rank r's send lands at r*count_per_rank.
 * In place on root: send == recv + root*count_per_rank. */
int b200mpi_gather(const void* send, void* recv, size_t count_per_rank, int dtype, int root, int memkind);
/* send (root only, may be NULL elsewhere) holds size()*count_per_rank; block r goes to rank r's recv.
 * In place on root: recv == send + root*count_per_rank. */
int b200mpi_scatter(const void* send, void* recv, size_t count_per_rank, int dtype, int root, int memkind);
/* counts[size()]: the same table on every rank (a rank whose table differs gets B200MPI_ERR_PEER, as
 * do all others).  Blocks are packed in rank order: displacement of rank r = counts[0] + ... +
 * counts[r-1] elements.  Any count may be 0.  In place: gatherv on root send == recv + displ[root],
 * scatterv on root recv == send + displ[root], allgatherv send == recv + displ[rank()].  Buffers
 * that are not in the b200mpi_alloc heap are staged whole through it (B200MPI_ERR_NOMEM if too big). */
int b200mpi_gatherv(const void* send, void* recv, const size_t* counts, int dtype, int root, int memkind);
int b200mpi_scatterv(const void* send, void* recv, const size_t* counts, int dtype, int root, int memkind);
int b200mpi_allgatherv(const void* send, void* recv, const size_t* counts, int dtype, int memkind);
/* send holds sum(send_counts) elements: block j (send_counts[j] elements, packed in rank order)
 * goes to rank j.  recv holds sum(recv_counts) elements: the block from rank r lands at
 * recv_counts[0] + ... + recv_counts[r-1].  recv_counts[r] on rank j must equal send_counts[j] on
 * rank r; ranks whose tables disagree get B200MPI_ERR_PEER, all of them, with no buffer touched.
 * Any count may be 0.  send == recv (in place) is B200MPI_ERR_ARG, as for alltoall.  Buffers outside
 * the b200mpi_alloc heap are staged whole through it (B200MPI_ERR_NOMEM if too big). */
int b200mpi_alltoallv(const void* send, const size_t* send_counts, void* recv, const size_t* recv_counts,
                      int dtype, int memkind);
/* Inclusive prefix reduction: recv on rank r = send_0 op send_1 op ... op send_r, element-wise,
 * combined left to right in rank order.  send == recv is in place. */
int b200mpi_scan(const void* send, void* recv, size_t count, int dtype, int op, int memkind);
/* Exclusive: recv on rank r >= 1 = send_0 op ... op send_{r-1}.  Rank 0's recv is not written
 * (it may be NULL there; in place, rank 0 keeps its input).  For both, buffers outside the
 * b200mpi_alloc heap are staged whole through it (B200MPI_ERR_NOMEM if too big). */
int b200mpi_exscan(const void* send, void* recv, size_t count, int dtype, int op, int memkind);
/* send holds sum(counts) elements; rank j receives op over r of rank r's block j, combined left to
 * right in rank order.  Block j starts at displacement counts[0] + ... + counts[j-1] of every send;
 * recv holds counts[rank()] elements and may be NULL where that is 0.  counts is the same table on
 * every rank (a rank whose table differs gets B200MPI_ERR_PEER, as do all others).  In place: recv ==
 * send + displ[rank()] (the form in-place Allgatherv completes).  Buffers outside the b200mpi_alloc
 * heap are staged whole through it (B200MPI_ERR_NOMEM if too big). */
int b200mpi_reduce_scatterv(const void* send, void* recv, const size_t* counts, int dtype, int op, int memkind);
/* Value-location reductions (MPI_MAXLOC / MPI_MINLOC).  An element is the 16-byte pair
 * struct { V val; int64_t loc; } with V = f32, f64 or i64 named by dtype (4 padding bytes follow an
 * f32 value); count counts pairs.  op B200MPI_MAX is MAXLOC, B200MPI_MIN is MINLOC (SUM and u8:
 * B200MPI_ERR_UNSUPPORTED).  Pairs are combined in rank order: a higher rank's pair replaces the
 * running one when its value is better, or equal with a smaller loc (signed).  Floats compare as
 * IEEE (-0 == +0), except that a NaN is better than every number for both ops and equal to every
 * NaN, so NaN propagates (MPI leaves NaN undefined).  The winning pair is copied whole, padding
 * included; of pairs equal in value and loc the lowest rank's wins, so the result does not depend on
 * the algorithm.  Buffers must be 8-byte aligned (B200MPI_ERR_ARG).  send == recv is in place;
 * reduce_loc writes root's recv only (it may be NULL elsewhere).  Buffers outside the b200mpi_alloc
 * heap are staged whole through it (B200MPI_ERR_NOMEM if too big). */
int b200mpi_allreduce_loc(const void* send, void* recv, size_t count, int dtype, int op, int memkind);
int b200mpi_reduce_loc(const void* send, void* recv, size_t count, int dtype, int op, int root, int memkind);
int b200mpi_barrier(void);

/* ---- one-sided communication: windows, Put / Get / Accumulate, fence (MPI-3 active target) ------ */

/* A window is [base, base + bytes) of this rank's b200mpi_alloc heap (anything else:
 * B200MPI_ERR_ARG); sizes may differ from rank to rank, and bytes == 0 with base == NULL is legal.
 * The library does not own the memory: freeing it while the window is live is erroneous (not
 * checked).  win_create is collective: every rank learns every rank's window, *win gets an id
 * handed out in call order and never reused; ranks whose ids differ, or whose peers refused their
 * arguments, get B200MPI_ERR_PEER and no window is created.  A freed or unknown id: B200MPI_ERR_ARG.
 * win_free is collective: a win_fence, then the id is dropped. */
int b200mpi_win_create(void* base, size_t bytes, int* win);
int b200mpi_win_free(int win);
/* Collective: every Put and Accumulate any rank issued into this window before its fence is visible
 * to the target once the target's win_fence returns, and every Get issued after a fence reads what
 * was there at that fence.  A fence on another window, or against b200mpi_barrier, ends as
 * B200MPI_ERR_PEER on every rank.  Within one fence epoch, a location written by one rank and read
 * or written by another (the target's own kernels and copies included, Put against Accumulate, and
 * Accumulates with different ops) is undefined, as in MPI. */
int b200mpi_win_fence(int win);
/* count elements of dtype between origin (memkind) and element target_disp of rank target's window:
 * (target_disp + count) * element size must fit in it (B200MPI_ERR_ARG).  Blocking: each returns once
 * origin may be reused; get's origin then holds the data.  Not collective (only the origin rank
 * calls them, on its collective thread) and they take no barrier epoch.  count == 0 returns 0 and
 * does nothing; a NULL origin with count > 0, a target out of range or an unknown dtype is
 * B200MPI_ERR_ARG.  Origins outside the heap are staged whole through it (B200MPI_ERR_NOMEM if too
 * big).  Put and Get take any alignment. */
int b200mpi_put(const void* origin, size_t count, int dtype, int target, size_t target_disp, int win, int memkind);
int b200mpi_get(void* origin, size_t count, int dtype, int target, size_t target_disp, int win, int memkind);
/* target[e] = target[e] op origin[e], each element an atomic read-modify-write at system scope, so
 * concurrent Accumulates with the same dtype and op on overlapping elements, from any ranks, combine
 * in some order.  dtype f32, f64 or i64 (u8: B200MPI_ERR_UNSUPPORTED); op SUM, MAX, MIN or REPLACE
 * (an element-wise atomic store of origin; NO_OP or unknown: B200MPI_ERR_ARG); the target element address must be a multiple of the element size
 * (B200MPI_ERR_ARG).  i64 SUM wraps; i64 MAX and MIN are exact; f64 SUM is one round-to-nearest add
 * per contribution, in an unspecified order.  f32 SUM flushes subnormals: on sm_90a an f32 atomic add
 * turns a subnormal input or result into zero of the same sign, unlike Allreduce, which keeps
 * subnormals.  f32 and f64 MAX and MIN apply b > a ? b : a (a = the target's value), so the result
 * does not depend on the order except for NaNs (a NaN in the target stays, a NaN contribution is
 * dropped) and zeros of mixed sign. */
int b200mpi_accumulate(const void* origin, size_t count, int dtype, int op, int target, size_t target_disp, int win, int memkind);

/* ---- one-sided communication, passive target: window locks and atomic fetches (MPI-3) ----------- */
/* Every call below is blocking, is not collective, takes no barrier epoch, and runs on the caller's
 * collective thread, like Put, Get and Accumulate.
 *
 * win_lock blocks until this rank holds the lock on rank target's window (target may be this rank).
 * B200MPI_LOCK_EXCLUSIVE excludes every other holder; B200MPI_LOCK_SHARED excludes only exclusive
 * holders.  There is no fairness: a steady stream of shared holders can starve an exclusive one (MPI
 * promises none either).  Not granted within the watchdog_ms knob: B200MPI_ERR_TIMEOUT, and nothing
 * is held.  B200MPI_ERR_ARG: an unknown or freed window, a bad lock type, a target out of range, or
 * a second lock on the same (target, win) by this rank.  win_unlock releases it (B200MPI_ERR_ARG if
 * this rank does not hold it).
 * Ordering: every RMA call completes before it returns, so everything this rank did to the target's
 * window before win_unlock is visible to the next rank that acquires that lock, of either type; there
 * is no separate flush call.  The target's own kernels and copies that touch its window must hold the
 * lock too, as MPI requires.  Put, Get and Accumulate work with or without locks.
 * Locks and fences do not mix on one window: win_fence or win_free by a rank that holds a lock on
 * that window returns B200MPI_ERR_ARG there and B200MPI_ERR_PEER on every other rank (in a world of
 * one: B200MPI_ERR_ARG, nothing launched); the window stays live and the lock held, and after the
 * unlock the next fence works. */
int b200mpi_win_lock(int lock_type, int target, int win);
int b200mpi_win_unlock(int target, int win);
/* result[e] = the target element's previous value, then target[e] = target[e] op origin[e], each
 * element one atomic read-modify-write at system scope: atomic with respect to Accumulate,
 * Get_accumulate, Fetch_and_op and Compare_and_swap on the same element with the same dtype, whatever
 * their ops, but not with respect to Put or Get (as in MPI).  dtype f32, f64 or i64 (u8:
 * B200MPI_ERR_UNSUPPORTED); op SUM, MAX, MIN, REPLACE (target = origin) or NO_OP (target unchanged,
 * origin may be NULL); anything else B200MPI_ERR_ARG.  The element rules are those of Accumulate (i64
 * SUM wraps, f32 SUM flushes subnormal inputs and results to zero of the same sign, float MAX and
 * MIN apply b > a ? b : a and b < a ? b : a); the fetched value is always the target's exact previous
 * bits.  Target range and alignment checks are those of Accumulate.  result holds count elements in
 * origin's memkind; result == origin is in place, any other overlap is B200MPI_ERR_ARG.  Origins and
 * results outside the heap, or heap pointers off element alignment, are staged whole (origin through
 * staging block 0, result through block 1; B200MPI_ERR_NOMEM if that does not fit). */
int b200mpi_get_accumulate(const void* origin, void* result, size_t count, int dtype, int op,
                           int target, size_t target_disp, int win, int memkind);
/* get_accumulate of one element, with origin and result host pointers to one element each (no
 * memkind; origin may be NULL for NO_OP).  The latency call: exactly one kernel launch and no staging
 * copies. */
int b200mpi_fetch_and_op(const void* origin, void* result, int dtype, int op,
                         int target, size_t target_disp, int win);
/* i64 only (f32, f64, u8: B200MPI_ERR_UNSUPPORTED): *result = the target element's old value, and
 * *origin is stored there if that old value equals *compare; one atomic at system scope.  Host
 * pointers to one element each, one kernel launch. */
int b200mpi_compare_and_swap(const void* origin, const void* compare, void* result, int dtype,
                             int target, size_t target_disp, int win);

/* ---- one-sided communication, generalized active target (MPI-3 post / start / complete / wait) --- */
/* A group is `count` distinct ranks in [0, size()); it may include this rank, and count == 0 is legal
 * (ranks may be NULL then).
 * None of these calls is collective or takes a barrier epoch.  Each runs on the caller's collective thread.
 *
 * win_start blocks until every target in its group has posted an exposure epoch that includes this
 * rank; then Put, Get and Accumulate to those targets are safe with no further waiting.  If a target
 * has not posted within the watchdog_ms knob: B200MPI_ERR_TIMEOUT, and no access epoch is open; the
 * posts that did arrive are not consumed, so a later win_start still sees them.  win_wait blocks until
 * every origin of the post's group has called win_complete for this epoch; if that does not happen
 * within watchdog_ms: B200MPI_ERR_TIMEOUT, and the exposure epoch stays open, so win_wait or win_test
 * may be called again.  win_test checks once and never waits.  An empty group opens and closes its
 * epoch without launching anything.
 * Ordering: every Put and Accumulate an origin issued between its win_start and its win_complete is
 * visible to the target, its own later kernels and copies included, once its win_wait returns (or
 * win_test sets *flag = 1).  A Get issued after win_start reads what the target's window held when
 * it called win_post.  The target's own writes to its window must be complete before win_post, and it
 * must not change the window locally between win_post and win_wait, as MPI requires.  Put, Get and
 * Accumulate are unchanged: they work inside or outside any epoch and do not check membership.
 * Errors (B200MPI_ERR_ARG, nothing launched): an unknown or freed window; a group with a NULL pointer
 * and count > 0, a negative count, count > size(), a rank out of range or a rank twice; win_post while
 * this rank's exposure epoch on the window is open; win_start while its access epoch is open;
 * win_complete with no access epoch open; win_wait or win_test with no exposure epoch open, or
 * win_test with a NULL flag.
 * Fences and locks: win_fence or win_free by a rank with an access or exposure epoch open on that
 * window returns B200MPI_ERR_ARG there and B200MPI_ERR_PEER on every other rank (in a world of one:
 * B200MPI_ERR_ARG, nothing launched), as under a held lock; the window stays live and the epoch open.
 * Locks and these epochs on one window are independent: both may be used, in turn or at once.
 * Erroneous programs: a target that posts to an origin which never starts on it (erroneous in MPI
 * too) only makes that target's win_wait time out; its exposure epoch stays open, so that rank's
 * win_fence and win_free of the window keep failing, until the origin starts and completes. */
int b200mpi_win_post(const int* origins, int count, int win);   /* open an exposure epoch to `origins`; does not block */
int b200mpi_win_start(const int* targets, int count, int win);  /* open an access epoch; blocks until every target has posted to this rank */
int b200mpi_win_complete(int win);                              /* close the access epoch: tells each target this rank is done */
int b200mpi_win_wait(int win);                                  /* close the exposure epoch: blocks until every origin has completed */
int b200mpi_win_test(int win, int* flag);                       /* win_wait without blocking: *flag = 1 and the epoch closed, or 0 and still open */

/* Enqueue-only forms on the library stream (DEVICE memkind only). */
int b200mpi_bcast_async(void* buf, size_t count, int dtype, int root);
int b200mpi_allreduce_async(const void* send, void* recv, size_t count, int dtype, int op);
int b200mpi_allgather_async(const void* send, void* recv, size_t count_per_rank, int dtype);
int b200mpi_reduce_scatter_async(const void* send, void* recv, size_t count_per_rank, int dtype, int op);
int b200mpi_stream_sync(void); /* waits and reports device-side watchdog errors */

/* ---- tuning / measurement ------------------------------------------------------------------ */

int b200mpi_set_algo(int coll, int algo); /* force an algorithm (benches, tests) */
int b200mpi_get_algo(int coll, size_t count, int dtype); /* what AUTO resolves to (>=1) or <0 */
int b200mpi_set_max_blocks(int blocks); /* cap grid size (0 = default: SMs x occupancy) */
/* Tuning knobs for sweeps: "twoshot_unroll" (0|1), "nvls_unroll" (1|2|4|8), "nvls_min_ranks",
 * "nvls_max_blocks", "oneshot_max_bytes", "ll_max_bytes", "stage_chunk", "pipe_min_bytes",
 * "pipe_chunk_bytes", "bounce_chunk_bytes", "host_threads", "own_block_bytes",
 * "hybrid_p2p_permille", "hybrid_p2p_blocks", "hybrid_min_bytes", "bcast_nvls2", "bcast_nvls_min",
 * "allgather_nvls_min", "host_register" (pin pageable host slices in place, cached; 0 drops the cache),
 * "p2p_fast" (host-slice Send/Receive through mapped pinned buffers), "watchdog_ms". */
int b200mpi_set_param(const char* name, int64_t value);
/* Reads every knob above, and these read-only values: "sm_count", "shared_device", "epoch" (the barrier
 * epoch the next launch takes) and "ll_seq" (the last LL Allreduce sequence number issued). */
int b200mpi_get_param(const char* name, int64_t* value);
/* cudaStream_t used for collectives; set NULL to restore the library's own stream. */
int b200mpi_get_stream(void** stream);
int b200mpi_set_stream(void* stream);
/* CUDA-event stopwatch on the collective stream. */
int b200mpi_timer_start(void);
int b200mpi_timer_stop(float* ms); /* synchronises; elapsed since timer_start */
/* Measured bound of the host-slice paths: pinned host <-> device-heap copy rates of this rank's GPU,
 * GB/s (1e9): H2D alone, D2H alone, and per direction with both running at once. */
int b200mpi_pcie_probe(size_t bytes, int iters, double* h2d_gbs, double* d2h_gbs, double* bidir_gbs);
/* Raw NVLink rates of the library's copy kernel between neighbouring ranks (collective call).
 * mode 0: every rank pulls `bytes` from rank+1; 1: every rank pushes to rank+1; 2 / 3: only rank 0
 * pulls from / pushes to rank 1; 4: every rank pulls and pushes at once.  *ms: device time per iteration. */
int b200mpi_link_probe(size_t bytes, int mode, int iters, float* ms);
/* Number of kernels this library has launched since init. */
int64_t b200mpi_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200MPI_H_ */
