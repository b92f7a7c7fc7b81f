// CPU-side checks of the Scan / Exscan facade of mpi_b200/cpp/mpi.hpp: a vector recv resized to
// len(send), the op and buffers passed through unchanged, and the answers before Init and from an
// implementation without these collectives.
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
  int scans = 0, exscans = 0;
  mpi::Op op = mpi::SUM;
  mpi::Buffer send{}, recv{};
  mpi::Error Scan(mpi::Buffer s, mpi::Buffer r, mpi::Op o) override { ++scans; send = s; recv = r; op = o; return {}; }
  mpi::Error Exscan(mpi::Buffer s, mpi::Buffer r, mpi::Op o) override { ++exscans; send = s; recv = r; op = o; return {}; }
};

int main() {
  // before Init the default implementation reports "not initialised"
  std::vector<double> x(5, 1.0), y;
  assert(mpi::Scan(x, &y).code == B200MPI_ERR_NOT_INIT);
  assert(mpi::Exscan(x, &y, mpi::MAX).code == B200MPI_ERR_NOT_INIT);

  Fake fake;
  mpi::Register(&fake);

  // a vector recv is resized to len(send); the op travels unchanged
  y.clear();
  assert(!mpi::Scan(x, &y, mpi::MIN) && y.size() == 5 && fake.scans == 1 && fake.op == mpi::MIN);
  assert(fake.send.ptr == x.data() && fake.recv.ptr == y.data() && fake.send.count == 5 && fake.recv.count == 5);
  assert(fake.send.dtype == B200MPI_F64 && fake.send.memkind == B200MPI_HOST);
  std::vector<int64_t> c(1, 42), d(9, 0);
  assert(!mpi::Exscan(c, &d) && d.size() == 1 && fake.exscans == 1 && fake.op == mpi::SUM && fake.send.dtype == B200MPI_I64);

  // device slices are passed as they are
  mpi::DeviceSlice<float> s(reinterpret_cast<float*>(4096), 8), r(reinterpret_cast<float*>(8192), 8);
  assert(!mpi::Scan(s, &r, mpi::MAX) && fake.send.memkind == B200MPI_DEVICE && fake.recv.ptr == r.data() && fake.recv.count == 8);
  assert(!mpi::Exscan(s, &r) && fake.exscans == 2 && fake.send.dtype == B200MPI_F32);

  // an implementation without these collectives says so
  Plain plain;
  mpi::mpier() = &plain;
  assert(mpi::Scan(x, &y).code == B200MPI_ERR_UNSUPPORTED);
  assert(mpi::Exscan(x, &y).code == B200MPI_ERR_UNSUPPORTED);
  printf("scan facade ok\n");
  return 0;
}
