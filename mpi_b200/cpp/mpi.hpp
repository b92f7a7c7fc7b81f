// mpi.hpp -- C++ host-side mirror of the reference's Go package `mpi`
// (/root/reference/mpi.go:56-182, flags.go:10-50) over the C ABI of include/b200mpi.h.
//
// The reference is compiled Go and this image has no Go toolchain, so the host layer above the
// C ABI is written in C++ with the same names, argument meaning and error behaviour; the Go shim
// that binds the same ABI is in go/ (see INTEGRATION.md).
//
//   Go                                         here
//   mpi.Init() error                           mpi::Error mpi::Init()
//   mpi.Finalize()                             void mpi::Finalize()
//   mpi.Rank() / mpi.Size()                    int mpi::Rank() / mpi::Size()
//   mpi.Send(data interface{}, dst, tag)       mpi::Error mpi::Send(const T& data, int dst, int tag)
//   mpi.Receive(&data, src, tag)               mpi::Error mpi::Receive(T* data, int src, int tag)   (resizes *data like gob)
//   mpi.Register(impl)                         void mpi::Register(Interface*)  (second call throws = panics, mpi.go:61-67)
//   flag.Parse() + mpi.Flag*                   mpi::ParseFlags(argc, argv) + mpi::Flag*
//   new: Recv, Bcast, Allreduce, Allgather, Barrier, ReduceScatter, Reduce, Alltoall, Isend/Wait,
//        Gather, Scatter, Gatherv, Scatterv, Allgatherv, Alltoallv, Scan, Exscan, ReduceScatterv,
//        AllreduceLoc, ReduceLoc (MAXLOC / MINLOC over mpi::ValLoc<V> pairs),
//        WinCreate -> mpi::Window with Put, Get, Accumulate, Fence, Free (one-sided, fence-synchronised)
//        and Lock, Unlock, GetAccumulate, FetchAndOp, CompareAndSwap (passive target)
//        and Post, Start, Complete, Wait, Test (generalized active target);
//        mpi::DeviceSlice<T> for heap-resident buffers
// `data` may be std::vector<double|float|int64_t|uint8_t>, std::string (sent as bytes, the
// "anything else is gob-encoded" path), or DeviceSlice<T>.
#pragma once
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/b200mpi.h"

namespace mpi {

// ---- error: nil-able like Go's `error` -----------------------------------------------------------
struct Error {
  int code = 0;
  std::string msg;
  explicit operator bool() const { return code != 0; } // `if (err)` reads like `if err != nil`
  const std::string& String() const { return msg; }
};
struct TagExists : Error { // mpi.go:174-182
  int Tag = 0;
};
inline Error make_error(int rc) {
  Error e;
  if (rc != 0) {
    e.code = rc;
    e.msg = b200mpi_last_error();
  }
  return e;
}

enum Op { SUM = B200MPI_SUM, MAX = B200MPI_MAX, MIN = B200MPI_MIN,
          REPLACE = B200MPI_REPLACE, NO_OP = B200MPI_NO_OP }; // REPLACE and NO_OP: one-sided calls only
enum LockType { LOCK_EXCLUSIVE = B200MPI_LOCK_EXCLUSIVE, LOCK_SHARED = B200MPI_LOCK_SHARED };
using Raw = std::vector<uint8_t>; // mpi.go:75

template <typename T> struct dtype_of;
template <> struct dtype_of<uint8_t> { static constexpr int value = B200MPI_U8; };
template <> struct dtype_of<char> { static constexpr int value = B200MPI_U8; };
template <> struct dtype_of<int64_t> { static constexpr int value = B200MPI_I64; };
template <> struct dtype_of<long long> { static constexpr int value = B200MPI_I64; };
template <> struct dtype_of<float> { static constexpr int value = B200MPI_F32; };
template <> struct dtype_of<double> { static constexpr int value = B200MPI_F64; };

// The element of AllreduceLoc / ReduceLoc (MPI's MAXLOC / MINLOC pairs): 16 bytes for V = float,
// double and int64_t.  It has no dtype_of, so no other call takes it.
template <typename V> struct ValLoc {
  V val;
  int64_t loc;
};
static_assert(sizeof(ValLoc<float>) == 16 && sizeof(ValLoc<double>) == 16 && sizeof(ValLoc<int64_t>) == 16, "pair layout");

// Memory from the rank's peer-mapped device heap: collectives and Send/Receive use it in place.
template <typename T>
class DeviceSlice {
 public:
  DeviceSlice() = default;
  explicit DeviceSlice(size_t count) : n_(count), own_(true) {
    void* p = nullptr;
    if (b200mpi_alloc(count * sizeof(T), &p) != 0) throw std::runtime_error(b200mpi_last_error());
    p_ = static_cast<T*>(p);
  }
  DeviceSlice(T* p, size_t count) : p_(p), n_(count), own_(false) {}
  DeviceSlice(const DeviceSlice&) = delete;
  DeviceSlice& operator=(const DeviceSlice&) = delete;
  DeviceSlice(DeviceSlice&& o) noexcept : p_(o.p_), n_(o.n_), own_(o.own_) { o.p_ = nullptr; o.own_ = false; }
  ~DeviceSlice() { if (own_ && p_) b200mpi_free(p_); }
  T* data() const { return p_; }
  size_t size() const { return n_; }
  DeviceSlice Sub(size_t lo, size_t hi) const { return DeviceSlice(p_ + lo, hi - lo); } // s[lo:hi]
  Error CopyFromHost(const std::vector<T>& h) { return make_error(b200mpi_memcpy(p_, h.data(), std::min(h.size(), n_) * sizeof(T), 0)); }
  Error CopyToHost(std::vector<T>* h) const { h->resize(n_); return make_error(b200mpi_memcpy(h->data(), p_, n_ * sizeof(T), 1)); }

 private:
  T* p_ = nullptr;
  size_t n_ = 0;
  bool own_ = false;
};

// ---- flags.go ---------------------------------------------------------------------------------------
inline std::string FlagAddr;
inline std::vector<std::string> FlagAllAddrs; // AddrsFlag: comma split, appends (flags.go:22-27)
inline int64_t FlagInitTimeout = 0;           // DurationFlag, nanoseconds
inline std::string FlagProtocol = "tcp";
inline std::string FlagPassword;
inline int FlagGpu = -1; // additive: -mpi-gpu

// time.ParseDuration subset used by -mpi-inittimeout ("300ms", "1.5s", "2m", "1h2m3s"); false if malformed
inline bool ParseDuration(const std::string& s, int64_t* ns) {
  if (s == "0") { *ns = 0; return true; }
  size_t i = 0;
  double sign = 1, total = 0;
  if (i < s.size() && (s[i] == '+' || s[i] == '-')) { if (s[i] == '-') sign = -1; ++i; }
  if (i >= s.size()) return false;
  while (i < s.size()) {
    size_t j = i;
    while (j < s.size() && (isdigit((unsigned char)s[j]) || s[j] == '.')) ++j;
    if (j == i) return false;
    double v = atof(s.substr(i, j - i).c_str());
    size_t k = j;
    while (k < s.size() && !isdigit((unsigned char)s[k]) && s[k] != '.') ++k;
    std::string u = s.substr(j, k - j);
    double mul;
    if (u == "ns") mul = 1; else if (u == "us" || u == "\xC2\xB5s") mul = 1e3; else if (u == "ms") mul = 1e6;
    else if (u == "s") mul = 1e9; else if (u == "m") mul = 60e9; else if (u == "h") mul = 3600e9; else return false;
    total += v * mul;
    i = k;
  }
  *ns = (int64_t)(sign * total + (sign * total >= 0 ? 0.5 : -0.5));
  return true;
}

// flag.Parse(): consumes the -mpi-* flags (one or two dashes, "-f v" or "-f=v"), returns the rest.
inline std::vector<std::string> ParseFlags(int argc, char** argv) {
  std::vector<std::string> rest;
  for (int i = 1; i < argc; ++i) {
    std::string a = argv[i];
    std::string name = a;
    while (!name.empty() && name[0] == '-') name.erase(0, 1);
    const bool is_flag = a.size() > 1 && a[0] == '-' && name.rfind("mpi-", 0) == 0;
    if (!is_flag) { rest.push_back(a); continue; }
    std::string value;
    size_t eq = name.find('=');
    if (eq != std::string::npos) { value = name.substr(eq + 1); name = name.substr(0, eq); }
    else if (i + 1 < argc) value = argv[++i];
    else throw std::runtime_error("flag needs an argument: -" + name);
    if (name == "mpi-addr") FlagAddr = value;
    else if (name == "mpi-alladdr") {
      size_t start = 0;
      for (;;) {
        size_t c = value.find(',', start);
        FlagAllAddrs.push_back(value.substr(start, c == std::string::npos ? std::string::npos : c - start));
        if (c == std::string::npos) break;
        start = c + 1;
      }
    } else if (name == "mpi-inittimeout") { if (!ParseDuration(value, &FlagInitTimeout)) throw std::runtime_error("invalid duration " + value); }
    else if (name == "mpi-protocol") FlagProtocol = value;
    else if (name == "mpi-password") FlagPassword = value;
    else if (name == "mpi-gpu") FlagGpu = atoi(value.c_str());
    else rest.push_back(a);
  }
  return rest;
}

// ---- mpi.Interface (mpi.go:163-170) + the optional collective upgrade (mpi.go:69-71) ---------------
struct Buffer { // what `data interface{}` is lowered to
  void* ptr;
  size_t count;
  int dtype;
  int memkind;
};
struct Interface {
  virtual ~Interface() = default;
  virtual Error Init() = 0;
  virtual void Finalize() = 0;
  virtual int Rank() = 0;
  virtual int Size() = 0;
  virtual Error Send(Buffer data, int destination, int tag) = 0;
  virtual Error Receive(Buffer data, size_t* count_out, int source, int tag) = 0;
  // collectives: default "not supported", like an implementation that is no AllReducer
  virtual Error Bcast(Buffer, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Bcast"; return e; }
  virtual Error Allreduce(Buffer, Buffer, Op) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Allreduce"; return e; }
  virtual Error Allgather(Buffer, Buffer) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Allgather"; return e; }
  virtual Error Barrier() { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Barrier"; return e; }
  virtual Error ReduceScatter(Buffer, Buffer, Op) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no ReduceScatter"; return e; }
  virtual Error Reduce(Buffer, Buffer, Op, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Reduce"; return e; }
  virtual Error Alltoall(Buffer, Buffer) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Alltoall"; return e; }
  // prefix reductions in rank order; Exscan leaves rank 0's recv unwritten (it may be empty there)
  virtual Error Scan(Buffer, Buffer, Op) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Scan"; return e; }
  virtual Error Exscan(Buffer, Buffer, Op) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Exscan"; return e; }
  // rooted and variable-count collectives: counts[Size()] is the same table on every rank
  virtual Error Gather(Buffer, Buffer, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Gather"; return e; }
  virtual Error Scatter(Buffer, Buffer, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Scatter"; return e; }
  virtual Error Gatherv(Buffer, Buffer, const size_t*, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Gatherv"; return e; }
  virtual Error Scatterv(Buffer, Buffer, const size_t*, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Scatterv"; return e; }
  virtual Error Allgatherv(Buffer, Buffer, const size_t*) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Allgatherv"; return e; }
  // send_counts / recv_counts[Size()]: this rank's row and column of the exchange (they differ from rank to rank)
  virtual Error Alltoallv(Buffer, const size_t*, Buffer, const size_t*) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Alltoallv"; return e; }
  // counts[Size()] is the same table on every rank: rank j receives the reduction of block j
  virtual Error ReduceScatterv(Buffer, Buffer, const size_t*, Op) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no ReduceScatterv"; return e; }
  // MAXLOC (MAX) / MINLOC (MIN) over ValLoc pairs, whose value type is the Buffer's dtype
  virtual Error AllreduceLoc(Buffer, Buffer, Op) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no AllreduceLoc"; return e; }
  virtual Error ReduceLoc(Buffer, Buffer, Op, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no ReduceLoc"; return e; }
  // one-sided: a window of `bytes` at `base` of this rank's heap gets an id; Put / Get / Accumulate
  // move a Buffer to or from element `disp` of rank `target`'s window
  virtual Error WinCreate(void*, size_t, int*) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no WinCreate"; return e; }
  virtual Error WinFree(int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no WinFree"; return e; }
  virtual Error WinFence(int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no WinFence"; return e; }
  virtual Error Put(Buffer, int, size_t, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Put"; return e; }
  virtual Error Get(Buffer, int, size_t, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Get"; return e; }
  virtual Error Accumulate(Buffer, Op, int, size_t, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Accumulate"; return e; }
  // passive target: a lock on rank `target`'s window, and the fetching atomics (one element each for
  // FetchAndOp and CompareAndSwap, through host pointers of the dtype)
  virtual Error WinLock(int, int, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no WinLock"; return e; }
  virtual Error WinUnlock(int, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no WinUnlock"; return e; }
  virtual Error GetAccumulate(Buffer, Buffer, Op, int, size_t, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no GetAccumulate"; return e; }
  virtual Error FetchAndOp(const void*, void*, int, Op, int, size_t, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no FetchAndOp"; return e; }
  virtual Error CompareAndSwap(const void*, const void*, void*, int, int, size_t, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no CompareAndSwap"; return e; }
  // generalized active target: a group is (ranks, count); WinTest sets *flag to 1 or 0
  virtual Error WinPost(const int*, int, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no WinPost"; return e; }
  virtual Error WinStart(const int*, int, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no WinStart"; return e; }
  virtual Error WinComplete(int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no WinComplete"; return e; }
  virtual Error WinWait(int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no WinWait"; return e; }
  virtual Error WinTest(int, int*) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no WinTest"; return e; }
  // the Send/Wait pair the reference sketches and comments out (mpi.go:132-152)
  virtual Error Isend(Buffer, int, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Isend"; return e; }
  virtual Error Wait(int, int) { Error e; e.code = B200MPI_ERR_UNSUPPORTED; e.msg = "registered implementation has no Wait"; return e; }
};

// The H100 implementation; plays the role of `Network` (network.go:25-39): fields win over flags.
struct Cuda : Interface {
  std::string Addr;
  std::vector<std::string> Addrs;
  int64_t Timeout = 0;
  std::string Password;
  int Gpu = -1;
  Error Init() override {
    if (Password.empty()) Password = FlagPassword; // useFlags, network.go:69-90
    if (Timeout == 0) Timeout = FlagInitTimeout;
    if (Addr.empty()) Addr = FlagAddr;
    if (Addrs.empty()) Addrs = FlagAllAddrs;
    if (Gpu < 0) Gpu = FlagGpu;
    std::string csv;
    for (size_t i = 0; i < Addrs.size(); ++i) csv += (i ? "," : "") + Addrs[i];
    return make_error(b200mpi_init(Addr.c_str(), csv.c_str(), Password.c_str(), Timeout, Gpu));
  }
  void Finalize() override { b200mpi_finalize(); }
  int Rank() override { return b200mpi_rank(); }
  int Size() override { return b200mpi_size(); }
  Error Send(Buffer d, int destination, int tag) override { return make_error(b200mpi_send(d.ptr, d.count, d.dtype, destination, tag, d.memkind)); }
  Error Receive(Buffer d, size_t* n, int source, int tag) override { return make_error(b200mpi_recv(d.ptr, d.count, n, d.dtype, source, tag, d.memkind)); }
  Error Bcast(Buffer d, int root) override { return make_error(b200mpi_bcast(d.ptr, d.count, d.dtype, root, d.memkind)); }
  Error Allreduce(Buffer s, Buffer r, Op op) override { return make_error(b200mpi_allreduce(s.ptr, r.ptr, s.count, s.dtype, op, s.memkind)); }
  Error Allgather(Buffer s, Buffer r) override { return make_error(b200mpi_allgather(s.ptr, r.ptr, s.count, s.dtype, s.memkind)); }
  Error Barrier() override { return make_error(b200mpi_barrier()); }
  Error ReduceScatter(Buffer s, Buffer r, Op op) override { return make_error(b200mpi_reduce_scatter(s.ptr, r.ptr, r.count, s.dtype, op, s.memkind)); }
  Error Reduce(Buffer s, Buffer r, Op op, int root) override { return make_error(b200mpi_reduce(s.ptr, r.ptr, s.count, s.dtype, op, root, s.memkind)); }
  Error Alltoall(Buffer s, Buffer r) override { return make_error(b200mpi_alltoall(s.ptr, r.ptr, s.count / (size_t)(Size() > 0 ? Size() : 1), s.dtype, s.memkind)); }
  Error Scan(Buffer s, Buffer r, Op op) override { return make_error(b200mpi_scan(s.ptr, r.ptr, s.count, s.dtype, op, s.memkind)); }
  Error Exscan(Buffer s, Buffer r, Op op) override { return make_error(b200mpi_exscan(s.ptr, r.ptr, s.count, s.dtype, op, s.memkind)); }
  Error Gather(Buffer s, Buffer r, int root) override { return make_error(b200mpi_gather(s.ptr, r.ptr, s.count, s.dtype, root, s.memkind)); }
  Error Scatter(Buffer s, Buffer r, int root) override { return make_error(b200mpi_scatter(s.ptr, r.ptr, r.count, r.dtype, root, r.memkind)); }
  Error Gatherv(Buffer s, Buffer r, const size_t* counts, int root) override { return make_error(b200mpi_gatherv(s.ptr, r.ptr, counts, s.dtype, root, s.memkind)); }
  Error Scatterv(Buffer s, Buffer r, const size_t* counts, int root) override { return make_error(b200mpi_scatterv(s.ptr, r.ptr, counts, r.dtype, root, r.memkind)); }
  Error Allgatherv(Buffer s, Buffer r, const size_t* counts) override { return make_error(b200mpi_allgatherv(s.ptr, r.ptr, counts, s.dtype, s.memkind)); }
  Error Alltoallv(Buffer s, const size_t* sc, Buffer r, const size_t* rc) override { return make_error(b200mpi_alltoallv(s.ptr, sc, r.ptr, rc, s.dtype, s.memkind)); }
  Error ReduceScatterv(Buffer s, Buffer r, const size_t* counts, Op op) override { return make_error(b200mpi_reduce_scatterv(s.ptr, r.ptr, counts, s.dtype, op, s.memkind)); }
  Error AllreduceLoc(Buffer s, Buffer r, Op op) override { return make_error(b200mpi_allreduce_loc(s.ptr, r.ptr, s.count, s.dtype, op, s.memkind)); }
  Error ReduceLoc(Buffer s, Buffer r, Op op, int root) override { return make_error(b200mpi_reduce_loc(s.ptr, r.ptr, s.count, s.dtype, op, root, s.memkind)); }
  Error WinCreate(void* base, size_t bytes, int* win) override { return make_error(b200mpi_win_create(base, bytes, win)); }
  Error WinFree(int win) override { return make_error(b200mpi_win_free(win)); }
  Error WinFence(int win) override { return make_error(b200mpi_win_fence(win)); }
  Error Put(Buffer o, int target, size_t disp, int win) override { return make_error(b200mpi_put(o.ptr, o.count, o.dtype, target, disp, win, o.memkind)); }
  Error Get(Buffer o, int target, size_t disp, int win) override { return make_error(b200mpi_get(o.ptr, o.count, o.dtype, target, disp, win, o.memkind)); }
  Error Accumulate(Buffer o, Op op, int target, size_t disp, int win) override {
    return make_error(b200mpi_accumulate(o.ptr, o.count, o.dtype, op, target, disp, win, o.memkind));
  }
  Error WinLock(int type, int target, int win) override { return make_error(b200mpi_win_lock(type, target, win)); }
  Error WinUnlock(int target, int win) override { return make_error(b200mpi_win_unlock(target, win)); }
  Error GetAccumulate(Buffer o, Buffer r, Op op, int target, size_t disp, int win) override {
    return make_error(b200mpi_get_accumulate(o.ptr, r.ptr, r.count, r.dtype, op, target, disp, win, r.memkind));
  }
  Error FetchAndOp(const void* o, void* r, int dtype, Op op, int target, size_t disp, int win) override {
    return make_error(b200mpi_fetch_and_op(o, r, dtype, op, target, disp, win));
  }
  Error CompareAndSwap(const void* o, const void* c, void* r, int dtype, int target, size_t disp, int win) override {
    return make_error(b200mpi_compare_and_swap(o, c, r, dtype, target, disp, win));
  }
  Error WinPost(const int* origins, int count, int win) override { return make_error(b200mpi_win_post(origins, count, win)); }
  Error WinStart(const int* targets, int count, int win) override { return make_error(b200mpi_win_start(targets, count, win)); }
  Error WinComplete(int win) override { return make_error(b200mpi_win_complete(win)); }
  Error WinWait(int win) override { return make_error(b200mpi_win_wait(win)); }
  Error WinTest(int win, int* flag) override { return make_error(b200mpi_win_test(win, flag)); }
  Error Isend(Buffer d, int destination, int tag) override { return make_error(b200mpi_isend(d.ptr, d.count, d.dtype, destination, tag, d.memkind)); }
  Error Wait(int destination, int tag) override { return make_error(b200mpi_wait(destination, tag)); }
};

inline Interface*& mpier() { // var mpier Interface = &Network{}  (mpi.go:56)
  static Cuda default_impl;
  static Interface* cur = &default_impl;
  return cur;
}
inline void Register(Interface* impl) { // mpi.go:61-67
  static bool called = false;
  mpier() = impl;
  if (called) throw std::logic_error("register called more than once");
  called = true;
}

// ---- lowering `data` ---------------------------------------------------------------------------------
template <typename T> inline Buffer lower(const std::vector<T>& v) { return {const_cast<T*>(v.data()), v.size(), dtype_of<T>::value, B200MPI_HOST}; }
inline Buffer lower(const std::string& s) { return {const_cast<char*>(s.data()), s.size(), B200MPI_U8, B200MPI_HOST}; }
template <typename T> inline Buffer lower(const DeviceSlice<T>& d) { return {d.data(), d.size(), dtype_of<T>::value, B200MPI_DEVICE}; }
// pairs: count in pairs, dtype of the value
template <typename V> inline Buffer lower_loc(const std::vector<ValLoc<V>>& v) { return {const_cast<ValLoc<V>*>(v.data()), v.size(), dtype_of<V>::value, B200MPI_HOST}; }
template <typename V> inline Buffer lower_loc(const DeviceSlice<ValLoc<V>>& d) { return {d.data(), d.size(), dtype_of<V>::value, B200MPI_DEVICE}; }

// ---- the package functions (mpi.go:96-159) -----------------------------------------------------------
inline Error Init() { return mpier()->Init(); }
inline void Finalize() { mpier()->Finalize(); }
inline int Rank() { return mpier()->Rank(); }
inline int Size() { return mpier()->Size(); }

template <typename D> inline Error Send(const D& data, int destination, int tag) { return mpier()->Send(lower(data), destination, tag); }

// Receive resizes *data to the sent length (gob does that for the reference, network.go:597).
template <typename T> inline Error Receive(std::vector<T>* data, int source, int tag) {
  size_t n = 0;
  Error e = mpier()->Receive(lower(*data), &n, source, tag);
  if (e.code == B200MPI_ERR_TRUNCATE) { // still posted: grow and take it
    data->resize(n);
    e = mpier()->Receive(lower(*data), &n, source, tag);
  }
  if (!e) data->resize(n);
  return e;
}
inline Error Receive(std::string* data, int source, int tag) {
  if (data->size() < 256) data->resize(256);
  size_t n = 0;
  Error e = mpier()->Receive(lower(*data), &n, source, tag);
  if (e.code == B200MPI_ERR_TRUNCATE) { data->resize(n); e = mpier()->Receive(lower(*data), &n, source, tag); }
  if (!e) data->resize(n);
  return e;
}
template <typename T> inline Error Receive(DeviceSlice<T>* data, size_t* count, int source, int tag) { return mpier()->Receive(lower(*data), count, source, tag); }
template <typename D> inline Error Recv(D* data, int source, int tag) { return Receive(data, source, tag); }

template <typename T> inline Error Bcast(std::vector<T>* data, int root) { return mpier()->Bcast(lower(*data), root); }
template <typename T> inline Error Bcast(DeviceSlice<T>* data, int root) { return mpier()->Bcast(lower(*data), root); }
template <typename T> inline Error Allreduce(const std::vector<T>& send, std::vector<T>* recv, Op op = SUM) {
  recv->resize(send.size());
  return mpier()->Allreduce(lower(send), lower(*recv), op);
}
template <typename T> inline Error Allreduce(const DeviceSlice<T>& send, DeviceSlice<T>* recv, Op op = SUM) { return mpier()->Allreduce(lower(send), lower(*recv), op); }
template <typename T> inline Error Allgather(const std::vector<T>& send, std::vector<T>* recv) {
  recv->resize(send.size() * (size_t)Size());
  return mpier()->Allgather(lower(send), lower(*recv));
}
template <typename T> inline Error Allgather(const DeviceSlice<T>& send, DeviceSlice<T>* recv) { return mpier()->Allgather(lower(send), lower(*recv)); }
inline Error Barrier() { return mpier()->Barrier(); }

// send holds Size() blocks; rank j receives the reduction of block j (recv is resized to one block)
template <typename T> inline Error ReduceScatter(const std::vector<T>& send, std::vector<T>* recv, Op op = SUM) {
  recv->resize(send.size() / (size_t)Size());
  return mpier()->ReduceScatter(lower(send), lower(*recv), op);
}
template <typename T> inline Error ReduceScatter(const DeviceSlice<T>& send, DeviceSlice<T>* recv, Op op = SUM) { return mpier()->ReduceScatter(lower(send), lower(*recv), op); }
template <typename T> inline Error Reduce(const std::vector<T>& send, std::vector<T>* recv, Op op, int root) {
  if (Rank() == root) recv->resize(send.size());
  return mpier()->Reduce(lower(send), lower(*recv), op, root);
}
template <typename T> inline Error Alltoall(const std::vector<T>& send, std::vector<T>* recv) {
  recv->resize(send.size());
  return mpier()->Alltoall(lower(send), lower(*recv));
}

// Scan: rank r's recv = send_0 op ... op send_r (rank order).  Exscan: up to send_{r-1}; rank 0's
// recv is not written.  A vector recv is resized to len(send).
template <typename T> inline Error Scan(const std::vector<T>& send, std::vector<T>* recv, Op op = SUM) {
  recv->resize(send.size());
  return mpier()->Scan(lower(send), lower(*recv), op);
}
template <typename T> inline Error Scan(const DeviceSlice<T>& send, DeviceSlice<T>* recv, Op op = SUM) { return mpier()->Scan(lower(send), lower(*recv), op); }
template <typename T> inline Error Exscan(const std::vector<T>& send, std::vector<T>* recv, Op op = SUM) {
  recv->resize(send.size());
  return mpier()->Exscan(lower(send), lower(*recv), op);
}
template <typename T> inline Error Exscan(const DeviceSlice<T>& send, DeviceSlice<T>* recv, Op op = SUM) { return mpier()->Exscan(lower(send), lower(*recv), op); }

// Gather: root's recv is resized to Size() blocks of len(send).  Scatter: root's recv is resized to
// one block of send; elsewhere recv must already hold that block length.
template <typename T> inline Error Gather(const std::vector<T>& send, std::vector<T>* recv, int root) {
  if (Rank() == root) recv->resize(send.size() * (size_t)Size());
  return mpier()->Gather(lower(send), lower(*recv), root);
}
template <typename T> inline Error Gather(const DeviceSlice<T>& send, DeviceSlice<T>* recv, int root) { return mpier()->Gather(lower(send), lower(*recv), root); }
template <typename T> inline Error Scatter(const std::vector<T>& send, std::vector<T>* recv, int root) {
  if (Rank() == root && Size() > 0) recv->resize(send.size() / (size_t)Size());
  return mpier()->Scatter(lower(send), lower(*recv), root);
}
template <typename T> inline Error Scatter(const DeviceSlice<T>& send, DeviceSlice<T>* recv, int root) { return mpier()->Scatter(lower(send), lower(*recv), root); }

inline Error arg_error(const std::string& msg) { Error e; e.code = B200MPI_ERR_ARG; e.msg = msg; return e; }
// An empty *counts is filled with every rank's len(send) through one int64 Allgather; a given one
// must hold Size() entries with counts[Rank()] == len(send).
inline Error fill_counts(size_t mine, std::vector<size_t>* counts, const char* what) {
  const size_t n = (size_t)(Size() > 0 ? Size() : 0);
  if (counts->empty() && n > 0) {
    std::vector<int64_t> one(1, (int64_t)mine), all;
    Error e = Allgather(one, &all);
    if (e) return e;
    counts->assign(all.begin(), all.end());
  }
  if (n > 0 && counts->size() != n) return arg_error(std::string("mpi: ") + what + " counts must hold Size() entries");
  if (n > 0 && (*counts)[(size_t)Rank()] != mine) return arg_error(std::string("mpi: ") + what + " counts[Rank()] must equal len(send)");
  return {};
}
inline size_t sum_of(const std::vector<size_t>& c) { size_t s = 0; for (size_t x : c) s += x; return s; }

// Gatherv / Allgatherv: root's (every rank's) recv is resized to sum(counts), as Receive resizes.
template <typename T> inline Error Gatherv(const std::vector<T>& send, std::vector<T>* recv, int root, std::vector<size_t>* counts) {
  Error e = fill_counts(send.size(), counts, "Gatherv");
  if (e) return e;
  if (Rank() == root) recv->resize(sum_of(*counts));
  return mpier()->Gatherv(lower(send), lower(*recv), counts->data(), root);
}
template <typename T> inline Error Allgatherv(const std::vector<T>& send, std::vector<T>* recv, std::vector<size_t>* counts) {
  Error e = fill_counts(send.size(), counts, "Allgatherv");
  if (e) return e;
  recv->resize(sum_of(*counts));
  return mpier()->Allgatherv(lower(send), lower(*recv), counts->data());
}
// Scatterv: root passes the table; root always sends it with one small Bcast, so the other ranks
// may pass an empty *counts and learn it.  recv is resized to counts[Rank()].
template <typename T> inline Error Scatterv(const std::vector<T>& send, std::vector<T>* recv, std::vector<size_t>* counts, int root) {
  const size_t n = (size_t)(Size() > 0 ? Size() : 0);
  const bool is_root = Rank() == root;
  if (n > 0 && ((is_root || !counts->empty()) && counts->size() != n)) return arg_error("mpi: Scatterv counts must hold Size() entries (root must pass them)");
  if (n > 0 && is_root && sum_of(*counts) != send.size()) return arg_error("mpi: Scatterv send must hold sum(counts) elements on root");
  if (n > 0) {
    std::vector<int64_t> table(n, 0);
    if (is_root) table.assign(counts->begin(), counts->end());
    Error e = Bcast(&table, root);
    if (e) return e;
    if (counts->empty()) counts->assign(table.begin(), table.end()); // a table that differs from root's fails as B200MPI_ERR_PEER
    recv->resize((*counts)[(size_t)Rank()]);
  }
  return mpier()->Scatterv(lower(send), lower(*recv), counts->data(), root);
}

// Alltoallv: block j of send (send_counts[j] elements, packed in rank order) goes to rank j.  An empty
// *recv_counts is learnt through one int64 Alltoall of send_counts; *recv is resized to
// sum(*recv_counts), as Receive resizes.
template <typename T> inline Error Alltoallv(const std::vector<T>& send, const std::vector<size_t>& send_counts, std::vector<T>* recv,
                                             std::vector<size_t>* recv_counts) {
  const size_t n = (size_t)(Size() > 0 ? Size() : 0);
  if (n > 0 && send_counts.size() != n) return arg_error("mpi: Alltoallv send_counts must hold Size() entries");
  if (n > 0 && sum_of(send_counts) != send.size()) return arg_error("mpi: Alltoallv send must hold sum(send_counts) elements");
  if (n > 0 && recv_counts->empty()) {
    std::vector<int64_t> mine(send_counts.begin(), send_counts.end()), theirs;
    Error e = Alltoall(mine, &theirs);
    if (e) return e;
    recv_counts->assign(theirs.begin(), theirs.end());
  }
  if (n > 0 && recv_counts->size() != n) return arg_error("mpi: Alltoallv recv_counts must hold Size() entries");
  recv->resize(sum_of(*recv_counts));
  return mpier()->Alltoallv(lower(send), send_counts.data(), lower(*recv), recv_counts->data());
}

// ReduceScatterv: send holds sum(counts) elements; rank j receives op over every rank's block j, in
// rank order.  *recv is resized to counts[Rank()], as Allgatherv resizes.
template <typename T> inline Error ReduceScatterv(const std::vector<T>& send, std::vector<T>* recv, const std::vector<size_t>& counts, Op op = SUM) {
  const size_t n = (size_t)(Size() > 0 ? Size() : 0);
  if (n > 0 && counts.size() != n) return arg_error("mpi: ReduceScatterv counts must hold Size() entries");
  if (n > 0 && sum_of(counts) != send.size()) return arg_error("mpi: ReduceScatterv send must hold sum(counts) elements");
  if (n > 0) recv->resize(counts[(size_t)Rank()]);
  return mpier()->ReduceScatterv(lower(send), lower(*recv), counts.data(), op);
}
template <typename T> inline Error ReduceScatterv(const DeviceSlice<T>& send, DeviceSlice<T>* recv, const std::vector<size_t>& counts, Op op = SUM) {
  return mpier()->ReduceScatterv(lower(send), lower(*recv), counts.data(), op);
}

// AllreduceLoc: every rank's recv gets, pair by pair, the winner of MAXLOC (op MAX) or MINLOC (op
// MIN) in rank order: a better value, or an equal one with a smaller loc; NaN beats every number.
// ReduceLoc: root's recv only.  A vector recv is resized to len(send) (on root for ReduceLoc).
template <typename V> inline Error AllreduceLoc(const std::vector<ValLoc<V>>& send, std::vector<ValLoc<V>>* recv, Op op = MAX) {
  recv->resize(send.size());
  return mpier()->AllreduceLoc(lower_loc(send), lower_loc(*recv), op);
}
template <typename V> inline Error AllreduceLoc(const DeviceSlice<ValLoc<V>>& send, DeviceSlice<ValLoc<V>>* recv, Op op = MAX) {
  return mpier()->AllreduceLoc(lower_loc(send), lower_loc(*recv), op);
}
template <typename V> inline Error ReduceLoc(const std::vector<ValLoc<V>>& send, std::vector<ValLoc<V>>* recv, Op op, int root) {
  if (Rank() == root) recv->resize(send.size());
  return mpier()->ReduceLoc(lower_loc(send), lower_loc(*recv), op, root);
}
template <typename V> inline Error ReduceLoc(const DeviceSlice<ValLoc<V>>& send, DeviceSlice<ValLoc<V>>* recv, Op op, int root) {
  return mpier()->ReduceLoc(lower_loc(send), lower_loc(*recv), op, root);
}

// One-sided communication through a window of every rank's heap (WinCreate, collective).  Put, Get
// and Accumulate move the origin (a vector or DeviceSlice) to or from element `disp` of rank
// `target`'s window, counted in the origin's element type, and return once the origin may be reused
// (Get: holds the data).  Their writes are visible to the target after its next Fence, which every
// rank calls; Free is a Fence that also drops the window.  Accumulate (SUM, MAX, MIN, REPLACE over
// float, double and int64_t) is element-wise atomic; an f32 SUM flushes subnormals to zero (b200mpi.h).
// Passive target: Lock / Unlock one target's window without the other ranks; GetAccumulate (the
// result has the origin's type, length and storage, and may be the origin; NO_OP takes nullptr as
// origin), FetchAndOp and CompareAndSwap (int64_t) return the target's previous values atomically.
// Generalized active target: a target exposes its window to a group with Post and closes the epoch
// with Wait (or Test, which never blocks); an origin opens an access epoch with Start, which blocks
// until every target has posted to it, and closes it with Complete.  Only the ranks in the groups
// take part; what an origin put between Start and Complete is visible to the target once its Wait
// returns.  A rank must not Fence or Free a window it holds a lock or has an epoch open on.
class Window {
 public:
  int id = -1;
  Error Lock(int target, LockType type = LOCK_EXCLUSIVE) { return mpier()->WinLock(type, target, id); }
  Error Unlock(int target) { return mpier()->WinUnlock(target, id); }
  template <typename D, typename R> Error GetAccumulate(const D& origin, R* result, int target, size_t disp, Op op = SUM) {
    const Buffer o = lower(origin), r = lower(*result);
    if (o.dtype != r.dtype || o.count != r.count || o.memkind != r.memkind) {
      Error e;
      e.code = B200MPI_ERR_ARG;
      e.msg = "GetAccumulate: origin and result differ in element type, length or storage";
      return e;
    }
    return mpier()->GetAccumulate(o, r, op, target, disp, id);
  }
  template <typename R> Error GetAccumulate(std::nullptr_t, R* result, int target, size_t disp, Op op = NO_OP) {
    Buffer none = lower(*result);
    none.ptr = nullptr;
    return mpier()->GetAccumulate(none, lower(*result), op, target, disp, id);
  }
  template <typename T> Error FetchAndOp(T value, T* result, int target, size_t disp, Op op = SUM) {
    return mpier()->FetchAndOp(op == NO_OP ? nullptr : &value, result, dtype_of<T>::value, op, target, disp, id);
  }
  Error CompareAndSwap(int64_t value, int64_t compare, int64_t* result, int target, size_t disp) {
    return mpier()->CompareAndSwap(&value, &compare, result, B200MPI_I64, target, disp, id);
  }
  template <typename D> Error Put(const D& origin, int target, size_t disp) { return mpier()->Put(lower(origin), target, disp, id); }
  template <typename T> Error Get(std::vector<T>* origin, int target, size_t disp) { return mpier()->Get(lower(*origin), target, disp, id); }
  template <typename T> Error Get(DeviceSlice<T>* origin, int target, size_t disp) { return mpier()->Get(lower(*origin), target, disp, id); }
  template <typename D> Error Accumulate(const D& origin, int target, size_t disp, Op op = SUM) { return mpier()->Accumulate(lower(origin), op, target, disp, id); }
  Error Post(const std::vector<int>& origins) { return mpier()->WinPost(origins.data(), (int)origins.size(), id); }
  Error Start(const std::vector<int>& targets) { return mpier()->WinStart(targets.data(), (int)targets.size(), id); }
  Error Complete() { return mpier()->WinComplete(id); }
  Error Wait() { return mpier()->WinWait(id); }
  Error Test(bool* flag) { // *flag: the exposure epoch has ended (and is closed)
    int f = 0;
    Error e = mpier()->WinTest(id, &f);
    if (!e) *flag = f != 0;
    return e;
  }
  Error Fence() { return mpier()->WinFence(id); }
  Error Free() { return mpier()->WinFree(id); }
};
template <typename T> inline Error WinCreate(const DeviceSlice<T>& local, Window* win) { return mpier()->WinCreate(local.data(), local.size() * sizeof(T), &win->id); }
inline Error WinCreate(std::nullptr_t, Window* win) { return mpier()->WinCreate(nullptr, 0, &win->id); } // an empty window

template <typename D> inline Error Isend(const D& data, int destination, int tag) { return mpier()->Isend(lower(data), destination, tag); }
inline Error Wait(int destination, int tag) { return mpier()->Wait(destination, tag); }

} // namespace mpi
