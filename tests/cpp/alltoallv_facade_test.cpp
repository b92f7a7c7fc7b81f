// CPU-side checks of the Alltoallv facade of mpi_b200/cpp/mpi.hpp: the receiver resized to
// sum(recv_counts) the way Receive resizes, an empty recv_counts learnt through one int64 Alltoall,
// shape errors before any collective, and the answers before Init and from an implementation
// without Alltoallv.
#include <cassert>
#include <cstdio>
#include <cstring>

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
  int calls = 0, alltoalls = 0;
  size_t send_count = 0, recv_count = 0;
  std::vector<size_t> sent_table, recv_table;
  mpi::Error Alltoall(mpi::Buffer s, mpi::Buffer r) override { // what ranks 0, 1, 2 send to rank 1: {4, send_counts[1], 6}
    assert(s.dtype == B200MPI_I64 && s.count == 3 && r.count == 3);
    ++alltoalls;
    int64_t* out = static_cast<int64_t*>(r.ptr);
    out[0] = 4; out[1] = static_cast<int64_t*>(s.ptr)[1]; out[2] = 6;
    return {};
  }
  mpi::Error Alltoallv(mpi::Buffer s, const size_t* sc, mpi::Buffer r, const size_t* rc) override {
    ++calls; send_count = s.count; recv_count = r.count;
    sent_table.assign(sc, sc + 3);
    recv_table.assign(rc, rc + 3);
    return {};
  }
};

int main() {
  // before Init the default implementation reports "not initialised"
  std::vector<float> x(6, 1.f), y;
  std::vector<size_t> counts = {1, 2, 3}, none;
  assert(mpi::Alltoallv(x, counts, &y, &none).code == B200MPI_ERR_NOT_INIT);

  Fake fake;
  mpi::Register(&fake);

  // a given recv table: recv is resized to its sum, both tables reach the implementation
  std::vector<size_t> rc = {5, 0, 2};
  y.assign(100, 0.f);
  assert(!mpi::Alltoallv(x, counts, &y, &rc) && y.size() == 7 && fake.recv_count == 7 && fake.send_count == 6);
  assert(fake.sent_table == counts && fake.recv_table == rc && fake.alltoalls == 0);

  // shape errors never reach the implementation
  const int before = fake.calls;
  std::vector<size_t> short_table = {3, 3};
  assert(mpi::Alltoallv(x, short_table, &y, &rc).code == B200MPI_ERR_ARG);
  std::vector<size_t> wrong_sum = {1, 2, 2};
  assert(mpi::Alltoallv(x, wrong_sum, &y, &rc).code == B200MPI_ERR_ARG);
  assert(mpi::Alltoallv(x, counts, &y, &short_table).code == B200MPI_ERR_ARG);
  assert(fake.calls == before);

  // recv counts omitted: learnt with one Alltoall of send_counts
  std::vector<size_t> learnt;
  y.clear();
  assert(!mpi::Alltoallv(x, counts, &y, &learnt) && (learnt == std::vector<size_t>{4, 2, 6}) && y.size() == 12);
  assert(fake.alltoalls == 1 && fake.recv_table == learnt);

  // an implementation without Alltoallv says so
  Plain plain;
  mpi::mpier() = &plain;
  assert(mpi::Alltoallv(x, counts, &y, &rc).code == B200MPI_ERR_UNSUPPORTED);
  printf("alltoallv facade ok\n");
  return 0;
}
