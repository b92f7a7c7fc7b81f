// CPU-side checks of the Gather / Scatter / Gatherv / Scatterv / Allgatherv facade of
// mpi_b200/cpp/mpi.hpp: receivers resized the way Receive resizes, counts learnt through one
// Allgather (Bcast of root's table for Scatterv), shape errors before any collective, and the
// answers before Init and from an implementation without these collectives.
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
  int calls = 0, root = -9;
  size_t send_count = 0, recv_count = 0;
  std::vector<size_t> table;
  mpi::Error Allgather(mpi::Buffer s, mpi::Buffer r) override { // every rank's length: {2, len(send), 4}
    assert(s.dtype == B200MPI_I64 && s.count == 1 && r.count == 3);
    int64_t* out = static_cast<int64_t*>(r.ptr);
    out[0] = 2; out[1] = *static_cast<int64_t*>(s.ptr); out[2] = 4;
    return {};
  }
  mpi::Error Bcast(mpi::Buffer d, int) override { // root's table
    assert(d.dtype == B200MPI_I64 && d.count == 3);
    int64_t t[3] = {5, 6, 7};
    memcpy(d.ptr, t, sizeof t);
    return {};
  }
  mpi::Error note(mpi::Buffer s, mpi::Buffer r, const size_t* c, int rt) {
    ++calls; root = rt; send_count = s.count; recv_count = r.count;
    table.assign(c, c + (c ? 3 : 0));
    return {};
  }
  mpi::Error Gather(mpi::Buffer s, mpi::Buffer r, int rt) override { return note(s, r, nullptr, rt); }
  mpi::Error Scatter(mpi::Buffer s, mpi::Buffer r, int rt) override { return note(s, r, nullptr, rt); }
  mpi::Error Gatherv(mpi::Buffer s, mpi::Buffer r, const size_t* c, int rt) override { return note(s, r, c, rt); }
  mpi::Error Scatterv(mpi::Buffer s, mpi::Buffer r, const size_t* c, int rt) override { return note(s, r, c, rt); }
  mpi::Error Allgatherv(mpi::Buffer s, mpi::Buffer r, const size_t* c) override { return note(s, r, c, -1); }
};

int main() {
  // before Init the default implementation reports "not initialised" for every new entry
  std::vector<float> x(3, 1.f), y;
  std::vector<size_t> none;
  assert(mpi::Gather(x, &y, 0).code == B200MPI_ERR_NOT_INIT);
  assert(mpi::Scatter(x, &y, 0).code == B200MPI_ERR_NOT_INIT);
  assert(mpi::Gatherv(x, &y, 0, &none).code == B200MPI_ERR_NOT_INIT);
  assert(mpi::Scatterv(x, &y, &none, 0).code == B200MPI_ERR_NOT_INIT);
  assert(mpi::Allgatherv(x, &y, &none).code == B200MPI_ERR_NOT_INIT);

  Fake fake;
  mpi::Register(&fake);

  // Gather: only root's recv is resized
  y.clear();
  assert(!mpi::Gather(x, &y, 1) && y.size() == 9 && fake.recv_count == 9 && fake.root == 1);
  y.assign(2, 0.f);
  assert(!mpi::Gather(x, &y, 0) && y.size() == 2);
  // Scatter: root's recv becomes one block of send
  std::vector<float> big(12, 0.f);
  assert(!mpi::Scatter(big, &y, 1) && y.size() == 4 && fake.send_count == 12);

  // Gatherv with a table: resized to its sum on root; shape errors never reach the implementation
  std::vector<size_t> counts = {2, 3, 4};
  y.clear();
  assert(!mpi::Gatherv(x, &y, 1, &counts) && y.size() == 9 && fake.table == counts);
  const int before = fake.calls;
  std::vector<size_t> short_table = {3, 3};
  assert(mpi::Gatherv(x, &y, 1, &short_table).code == B200MPI_ERR_ARG);
  std::vector<size_t> wrong_mine = {2, 5, 4};
  assert(mpi::Gatherv(x, &y, 1, &wrong_mine).code == B200MPI_ERR_ARG);
  assert(mpi::Allgatherv(x, &y, &wrong_mine).code == B200MPI_ERR_ARG);
  assert(fake.calls == before);

  // counts omitted: learnt with one Allgather of the lengths
  std::vector<size_t> learnt;
  y.clear();
  assert(!mpi::Gatherv(x, &y, 1, &learnt) && learnt == counts && y.size() == 9);
  std::vector<size_t> learnt2;
  std::vector<float> z(100, 0.f);
  assert(!mpi::Allgatherv(x, &z, &learnt2) && learnt2 == counts && z.size() == 9 && fake.recv_count == 9);

  // Scatterv off root: the table comes from root's Bcast, recv is resized to this rank's block
  std::vector<size_t> from_root;
  std::vector<float> empty, r;
  assert(!mpi::Scatterv(empty, &r, &from_root, 0) && r.size() == 6 && (from_root == std::vector<size_t>{5, 6, 7}));
  // on root the table is required and must cover send
  std::vector<size_t> bad = {1, 1, 1};
  assert(mpi::Scatterv(big, &r, &bad, 1).code == B200MPI_ERR_ARG);
  std::vector<size_t> ok = {5, 6, 1};
  assert(!mpi::Scatterv(big, &r, &ok, 1) && r.size() == 6 && fake.table == ok);

  // an implementation without these collectives says so
  Plain plain;
  mpi::mpier() = &plain;
  assert(mpi::Gather(x, &y, 0).code == B200MPI_ERR_UNSUPPORTED);
  assert(mpi::Allgatherv(x, &y, &counts).code == B200MPI_ERR_UNSUPPORTED);
  printf("gather facade ok\n");
  return 0;
}
