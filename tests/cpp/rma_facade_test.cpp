// CPU-side checks of the one-sided facade of mpi_b200/cpp/mpi.hpp: WinCreate passes the slice's bytes
// (or an empty window) and keeps the id; Put, Get and Accumulate lower vectors and device slices with
// their dtype, count and memory kind and pass target, displacement, op and window id unchanged; Fence
// and Free reach the implementation with the id; the answers before Init and from an implementation
// without one-sided calls.
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
  int creates = 0, puts = 0, gets = 0, accs = 0, fences = 0, frees = 0, target = -1, win = -1;
  void* base = nullptr;
  size_t bytes = 0, disp = 0;
  mpi::Op op = mpi::MAX;
  mpi::Buffer origin{};
  mpi::Error WinCreate(void* b, size_t n, int* w) override { base = b; bytes = n; *w = 40 + creates++; return {}; }
  mpi::Error WinFree(int w) override { ++frees; win = w; return {}; }
  mpi::Error WinFence(int w) override { ++fences; win = w; return {}; }
  mpi::Error Put(mpi::Buffer o, int t, size_t d, int w) override { ++puts; origin = o; target = t; disp = d; win = w; return {}; }
  mpi::Error Get(mpi::Buffer o, int t, size_t d, int w) override { ++gets; origin = o; target = t; disp = d; win = w; return {}; }
  mpi::Error Accumulate(mpi::Buffer o, mpi::Op p, int t, size_t d, int w) override { ++accs; origin = o; op = p; target = t; disp = d; win = w; return {}; }
};

int main() {
  // before Init the default implementation reports "not initialised"
  mpi::Window w0;
  assert(mpi::WinCreate(nullptr, &w0).code == B200MPI_ERR_NOT_INIT && w0.id == -1);
  std::vector<double> x(5, 1.0);
  assert(w0.Put(x, 0, 0).code == B200MPI_ERR_NOT_INIT);
  assert(w0.Get(&x, 0, 0).code == B200MPI_ERR_NOT_INIT);
  assert(w0.Accumulate(x, 0, 0).code == B200MPI_ERR_NOT_INIT);
  assert(w0.Fence().code == B200MPI_ERR_NOT_INIT && w0.Free().code == B200MPI_ERR_NOT_INIT);

  Fake fake;
  mpi::Register(&fake);

  // WinCreate: the slice's bytes, or an empty window; the id is kept
  mpi::DeviceSlice<float> local(reinterpret_cast<float*>(4096), 10);
  mpi::Window w;
  assert(!mpi::WinCreate(local, &w) && w.id == 40 && fake.base == local.data() && fake.bytes == 40);
  mpi::Window e;
  assert(!mpi::WinCreate(nullptr, &e) && e.id == 41 && fake.base == nullptr && fake.bytes == 0);

  // Put / Get / Accumulate of vectors: host memory, the element type's dtype and count
  assert(!w.Put(x, 2, 7) && fake.puts == 1 && fake.origin.ptr == x.data() && fake.origin.count == 5);
  assert(fake.origin.dtype == B200MPI_F64 && fake.origin.memkind == B200MPI_HOST && fake.target == 2 && fake.disp == 7 && fake.win == 40);
  std::vector<int64_t> y(3);
  assert(!e.Get(&y, 0, 1) && fake.gets == 1 && fake.origin.ptr == y.data() && fake.origin.dtype == B200MPI_I64 && fake.win == 41);
  assert(fake.target == 0 && fake.disp == 1 && fake.origin.count == 3);
  assert(!w.Accumulate(y, 1, 9) && fake.accs == 1 && fake.op == mpi::SUM && fake.target == 1 && fake.disp == 9);
  std::vector<float> f(4);
  assert(!w.Accumulate(f, 2, 0, mpi::MIN) && fake.op == mpi::MIN && fake.origin.dtype == B200MPI_F32 && fake.origin.count == 4);

  // device slices are passed as they are
  mpi::DeviceSlice<double> d(reinterpret_cast<double*>(8192), 6);
  assert(!w.Put(d, 1, 3) && fake.origin.ptr == d.data() && fake.origin.memkind == B200MPI_DEVICE && fake.origin.count == 6);
  assert(!w.Get(&d, 2, 0) && fake.gets == 2 && fake.origin.memkind == B200MPI_DEVICE && fake.target == 2);
  assert(!w.Accumulate(d, 0, 4, mpi::MAX) && fake.accs == 3 && fake.op == mpi::MAX && fake.origin.dtype == B200MPI_F64);

  // Fence and Free carry the id
  assert(!e.Fence() && fake.fences == 1 && fake.win == 41);
  assert(!w.Free() && fake.frees == 1 && fake.win == 40);

  // an implementation without one-sided calls says so
  Plain plain;
  mpi::mpier() = &plain;
  mpi::Window p;
  assert(mpi::WinCreate(local, &p).code == B200MPI_ERR_UNSUPPORTED);
  assert(w.Put(x, 0, 0).code == B200MPI_ERR_UNSUPPORTED && w.Get(&x, 0, 0).code == B200MPI_ERR_UNSUPPORTED);
  assert(w.Accumulate(x, 0, 0).code == B200MPI_ERR_UNSUPPORTED);
  assert(w.Fence().code == B200MPI_ERR_UNSUPPORTED && w.Free().code == B200MPI_ERR_UNSUPPORTED);
  printf("rma facade ok\n");
  return 0;
}
