// CPU-side checks of the passive-target facade of mpi_b200/cpp/mpi.hpp: Lock and Unlock pass the lock
// type, target and window id; GetAccumulate lowers origin and result (vectors or device slices) and
// refuses a pair that differs in type, length or storage; NO_OP takes nullptr as its origin;
// FetchAndOp passes the element's dtype and a NULL origin for NO_OP; CompareAndSwap passes its three
// int64_t words; the answers before Init and from an implementation without passive-target calls.
#include <cassert>
#include <cstdio>

#include "../../mpi_b200/cpp/mpi.hpp"

struct Plain : mpi::Interface { // rank 1 of 3, no collectives
  mpi::Error Init() override { return {}; }
  void Finalize() override {}
  int Rank() override { return 1; }
  int Size() override { return 3; }
  mpi::Error Send(mpi::Buffer, int, int) override { return {}; }
  mpi::Error Receive(mpi::Buffer, size_t* n, int, int) override { *n = 0; return {}; }
};

struct Fake : Plain { // records what reaches the implementation
  int locks = 0, unlocks = 0, gas = 0, fops = 0, cases = 0, type = -1, target = -1, win = -1, dtype = -1;
  size_t disp = 0;
  mpi::Op op = mpi::MAX;
  mpi::Buffer origin{}, result{};
  const void* o = nullptr;
  const void* c = nullptr;
  void* r = nullptr;
  mpi::Error WinLock(int t, int tg, int w) override { ++locks; type = t; target = tg; win = w; return {}; }
  mpi::Error WinUnlock(int tg, int w) override { ++unlocks; target = tg; win = w; return {}; }
  mpi::Error GetAccumulate(mpi::Buffer og, mpi::Buffer rs, mpi::Op p, int tg, size_t d, int w) override {
    ++gas; origin = og; result = rs; op = p; target = tg; disp = d; win = w; return {};
  }
  mpi::Error FetchAndOp(const void* og, void* rs, int dt, mpi::Op p, int tg, size_t d, int w) override {
    ++fops; o = og; r = rs; dtype = dt; op = p; target = tg; disp = d; win = w;
    if (dt == B200MPI_F64) *(double*)rs = og ? *(const double*)og + 0.5 : -1.0;
    return {};
  }
  mpi::Error CompareAndSwap(const void* og, const void* cm, void* rs, int dt, int tg, size_t d, int w) override {
    ++cases; o = og; c = cm; r = rs; dtype = dt; target = tg; disp = d; win = w;
    *(int64_t*)rs = *(const int64_t*)og * 100 + *(const int64_t*)cm;
    return {};
  }
};

int main() {
  // before Init the default implementation reports "not initialised"
  mpi::Window w0;
  std::vector<double> x(5, 1.0), y(5);
  double dv = 0;
  int64_t iv = 0;
  assert(w0.Lock(0).code == B200MPI_ERR_NOT_INIT && w0.Unlock(0).code == B200MPI_ERR_NOT_INIT);
  assert(w0.GetAccumulate(x, &y, 0, 0).code == B200MPI_ERR_NOT_INIT);
  assert(w0.FetchAndOp(1.0, &dv, 0, 0).code == B200MPI_ERR_NOT_INIT);
  assert(w0.CompareAndSwap(1, 2, &iv, 0, 0).code == B200MPI_ERR_NOT_INIT);

  Fake fake;
  mpi::Register(&fake);
  mpi::Window w;
  w.id = 42;

  // Lock: exclusive by default, shared on request; Unlock carries target and id
  assert(!w.Lock(2) && fake.locks == 1 && fake.type == B200MPI_LOCK_EXCLUSIVE && fake.target == 2 && fake.win == 42);
  assert(!w.Lock(1, mpi::LOCK_SHARED) && fake.type == B200MPI_LOCK_SHARED && fake.target == 1);
  assert(!w.Unlock(0) && fake.unlocks == 1 && fake.target == 0 && fake.win == 42);

  // GetAccumulate of vectors: both buffers lowered, SUM by default
  assert(!w.GetAccumulate(x, &y, 1, 7) && fake.gas == 1 && fake.origin.ptr == x.data() && fake.result.ptr == y.data());
  assert(fake.result.count == 5 && fake.result.dtype == B200MPI_F64 && fake.result.memkind == B200MPI_HOST && fake.op == mpi::SUM);
  assert(fake.target == 1 && fake.disp == 7 && fake.win == 42);
  assert(!w.GetAccumulate(x, &x, 0, 0, mpi::REPLACE) && fake.origin.ptr == fake.result.ptr && fake.op == mpi::REPLACE); // in place
  // device slices; NO_OP without an origin
  mpi::DeviceSlice<int64_t> d(reinterpret_cast<int64_t*>(8192), 6), e(reinterpret_cast<int64_t*>(16384), 6);
  assert(!w.GetAccumulate(d, &e, 2, 3, mpi::MAX) && fake.result.memkind == B200MPI_DEVICE && fake.result.dtype == B200MPI_I64 && fake.op == mpi::MAX);
  assert(!w.GetAccumulate(nullptr, &e, 0, 1) && fake.gas == 4 && fake.origin.ptr == nullptr && fake.op == mpi::NO_OP && fake.result.ptr == e.data());
  // origin and result must agree: type, length, storage
  std::vector<float> f(5);
  std::vector<double> shorter(4);
  std::vector<int64_t> hosti(6);
  assert(w.GetAccumulate(x, &f, 0, 0).code == B200MPI_ERR_ARG);
  assert(w.GetAccumulate(x, &shorter, 0, 0).code == B200MPI_ERR_ARG);
  assert(w.GetAccumulate(d, &hosti, 0, 0).code == B200MPI_ERR_ARG && fake.gas == 4);

  // FetchAndOp: the value's dtype, the op, a NULL origin for NO_OP
  assert(!w.FetchAndOp(2.0, &dv, 1, 9) && fake.fops == 1 && fake.dtype == B200MPI_F64 && fake.op == mpi::SUM && dv == 2.5);
  assert(fake.r == &dv && fake.target == 1 && fake.disp == 9 && fake.win == 42);
  assert(!w.FetchAndOp(0.0, &dv, 0, 0, mpi::NO_OP) && fake.o == nullptr && dv == -1.0 && fake.op == mpi::NO_OP);
  float fv = 0;
  assert(!w.FetchAndOp(1.5f, &fv, 2, 1, mpi::MIN) && fake.dtype == B200MPI_F32 && fake.op == mpi::MIN && fake.r == &fv);
  assert(!w.FetchAndOp(int64_t(3), &iv, 2, 1, mpi::REPLACE) && fake.dtype == B200MPI_I64 && fake.op == mpi::REPLACE);

  // CompareAndSwap: value, compare and result as int64_t
  assert(!w.CompareAndSwap(7, -1, &iv, 2, 5) && fake.cases == 1 && fake.dtype == B200MPI_I64 && iv == 699);
  assert(fake.target == 2 && fake.disp == 5 && fake.win == 42 && fake.r == &iv);

  // an implementation without passive-target calls says so
  Plain plain;
  mpi::mpier() = &plain;
  assert(w.Lock(0).code == B200MPI_ERR_UNSUPPORTED && w.Unlock(0).code == B200MPI_ERR_UNSUPPORTED);
  assert(w.GetAccumulate(x, &y, 0, 0).code == B200MPI_ERR_UNSUPPORTED && w.GetAccumulate(nullptr, &y, 0, 0).code == B200MPI_ERR_UNSUPPORTED);
  assert(w.FetchAndOp(1.0, &dv, 0, 0).code == B200MPI_ERR_UNSUPPORTED);
  assert(w.CompareAndSwap(1, 2, &iv, 0, 0).code == B200MPI_ERR_UNSUPPORTED);
  printf("rma atomic facade ok\n");
  return 0;
}
