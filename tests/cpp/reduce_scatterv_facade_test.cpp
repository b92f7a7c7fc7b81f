// CPU-side checks of the ReduceScatterv facade of mpi_b200/cpp/mpi.hpp: a vector recv resized to
// counts[Rank()], the table, op and buffers passed through unchanged, the table checks, and the
// answers before Init and from an implementation without this collective.
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
  int calls = 0;
  mpi::Op op = mpi::SUM;
  mpi::Buffer send{}, recv{};
  const size_t* counts = nullptr;
  mpi::Error ReduceScatterv(mpi::Buffer s, mpi::Buffer r, const size_t* c, mpi::Op o) override {
    ++calls; send = s; recv = r; counts = c; op = o;
    return {};
  }
};

int main() {
  // before Init the default implementation reports "not initialised"
  std::vector<double> x(7, 1.0), y;
  const std::vector<size_t> table = {2, 4, 1};
  assert(mpi::ReduceScatterv(x, &y, table).code == B200MPI_ERR_NOT_INIT);

  Fake fake;
  mpi::Register(&fake);

  // a vector recv is resized to counts[Rank()]; table and op travel unchanged
  assert(!mpi::ReduceScatterv(x, &y, table, mpi::MIN) && y.size() == 4 && fake.calls == 1 && fake.op == mpi::MIN);
  assert(fake.send.ptr == x.data() && fake.send.count == 7 && fake.recv.ptr == y.data() && fake.recv.count == 4);
  assert(fake.counts == table.data() && fake.send.dtype == B200MPI_F64 && fake.send.memkind == B200MPI_HOST);
  std::vector<int64_t> c(3, 5), d(9, 0);
  const std::vector<size_t> zero_here = {3, 0, 0};
  assert(!mpi::ReduceScatterv(c, &d, zero_here) && d.empty() && fake.calls == 2 && fake.op == mpi::SUM && fake.send.dtype == B200MPI_I64);

  // the table is checked before the implementation is called
  std::vector<double> z;
  assert(mpi::ReduceScatterv(x, &z, std::vector<size_t>{3, 4}).code == B200MPI_ERR_ARG);    // not Size() entries
  assert(mpi::ReduceScatterv(x, &z, std::vector<size_t>{3, 4, 1}).code == B200MPI_ERR_ARG); // sum != len(send)
  assert(fake.calls == 2 && z.empty());

  // device slices are passed as they are
  mpi::DeviceSlice<float> s(reinterpret_cast<float*>(4096), 7), r(reinterpret_cast<float*>(8192), 4);
  assert(!mpi::ReduceScatterv(s, &r, table, mpi::MAX) && fake.calls == 3 && fake.send.memkind == B200MPI_DEVICE);
  assert(fake.recv.ptr == r.data() && fake.recv.count == 4 && fake.send.dtype == B200MPI_F32 && fake.op == mpi::MAX);

  // an implementation without this collective says so
  Plain plain;
  mpi::mpier() = &plain;
  assert(mpi::ReduceScatterv(x, &y, table).code == B200MPI_ERR_UNSUPPORTED);
  printf("reduce_scatterv facade ok\n");
  return 0;
}
