// CPU-side checks of the AllreduceLoc / ReduceLoc facade of mpi_b200/cpp/mpi.hpp: the ValLoc layout,
// vector recvs resized to len(send) (ReduceLoc: on root only), pairs lowered with the value's dtype
// and the pair count, op and root passed through unchanged, and the answers before Init and from an
// implementation without these collectives.
#include <cassert>
#include <cstddef>
#include <cstdio>

#include "../../mpi_b200/cpp/mpi.hpp"

static_assert(offsetof(mpi::ValLoc<float>, loc) == 8 && offsetof(mpi::ValLoc<double>, loc) == 8, "loc at byte 8");

struct Plain : mpi::Interface { // rank 1 of 3, no collectives
  mpi::Error Init() override { return {}; }
  void Finalize() override {}
  int Rank() override { return 1; }
  int Size() override { return 3; }
  mpi::Error Send(mpi::Buffer, int, int) override { return {}; }
  mpi::Error Receive(mpi::Buffer, size_t* n, int, int) override { *n = 0; return {}; }
};

struct Fake : Plain { // records what reaches the implementation
  int all = 0, rooted = 0, root = -1;
  mpi::Op op = mpi::SUM;
  mpi::Buffer send{}, recv{};
  mpi::Error AllreduceLoc(mpi::Buffer s, mpi::Buffer r, mpi::Op o) override {
    ++all; send = s; recv = r; op = o;
    return {};
  }
  mpi::Error ReduceLoc(mpi::Buffer s, mpi::Buffer r, mpi::Op o, int rt) override {
    ++rooted; send = s; recv = r; op = o; root = rt;
    return {};
  }
};

int main() {
  // before Init the default implementation reports "not initialised"
  std::vector<mpi::ValLoc<double>> x(5, mpi::ValLoc<double>{1.0, 7}), y;
  assert(mpi::AllreduceLoc(x, &y).code == B200MPI_ERR_NOT_INIT);
  assert(mpi::ReduceLoc(x, &y, mpi::MIN, 0).code == B200MPI_ERR_NOT_INIT);

  Fake fake;
  mpi::Register(&fake);

  // a vector recv is resized to len(send); the pair count, the value's dtype and the op travel
  assert(!mpi::AllreduceLoc(x, &y) && y.size() == 5 && fake.all == 1 && fake.op == mpi::MAX);
  assert(fake.send.ptr == x.data() && fake.send.count == 5 && fake.recv.ptr == y.data() && fake.recv.count == 5);
  assert(fake.send.dtype == B200MPI_F64 && fake.send.memkind == B200MPI_HOST);
  std::vector<mpi::ValLoc<float>> f(3), g;
  assert(!mpi::AllreduceLoc(f, &g, mpi::MIN) && g.size() == 3 && fake.send.dtype == B200MPI_F32 && fake.op == mpi::MIN);

  // ReduceLoc resizes on root only (this is rank 1)
  std::vector<mpi::ValLoc<int64_t>> a(4), b;
  assert(!mpi::ReduceLoc(a, &b, mpi::MAX, 0) && b.empty() && fake.rooted == 1 && fake.root == 0 && fake.send.dtype == B200MPI_I64);
  assert(fake.recv.count == 0 && fake.send.count == 4);
  assert(!mpi::ReduceLoc(a, &b, mpi::MIN, 1) && b.size() == 4 && fake.root == 1 && fake.op == mpi::MIN && fake.recv.ptr == b.data());

  // device slices are passed as they are
  mpi::DeviceSlice<mpi::ValLoc<float>> s(reinterpret_cast<mpi::ValLoc<float>*>(4096), 6), r(reinterpret_cast<mpi::ValLoc<float>*>(8192), 6);
  assert(!mpi::AllreduceLoc(s, &r, mpi::MAX) && fake.all == 3 && fake.send.memkind == B200MPI_DEVICE && fake.send.count == 6);
  assert(fake.recv.ptr == r.data() && fake.send.dtype == B200MPI_F32);
  assert(!mpi::ReduceLoc(s, &r, mpi::MIN, 2) && fake.rooted == 3 && fake.root == 2 && fake.recv.memkind == B200MPI_DEVICE);

  // an implementation without these collectives says so
  Plain plain;
  mpi::mpier() = &plain;
  assert(mpi::AllreduceLoc(x, &y).code == B200MPI_ERR_UNSUPPORTED);
  assert(mpi::ReduceLoc(x, &y, mpi::MAX, 0).code == B200MPI_ERR_UNSUPPORTED);
  printf("loc facade ok\n");
  return 0;
}
