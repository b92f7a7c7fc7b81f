// CPU-side checks of the generalized active-target facade of mpi_b200/cpp/mpi.hpp: Post and Start pass
// the group's ranks and size (an empty group too) and the window id; Complete and Wait pass the id;
// Test turns the implementation's flag into a bool and leaves it alone on an error; the answers
// before Init and from an implementation without these calls.
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
  int posts = 0, starts = 0, completes = 0, waits = 0, tests = 0, win = -1, count = -1, test_flag = 1;
  std::vector<int> group;
  mpi::Error WinPost(const int* r, int n, int w) override { ++posts; group.assign(r, r + n); count = n; win = w; return {}; }
  mpi::Error WinStart(const int* r, int n, int w) override { ++starts; group.assign(r, r + n); count = n; win = w; return {}; }
  mpi::Error WinComplete(int w) override { ++completes; win = w; return {}; }
  mpi::Error WinWait(int w) override { ++waits; win = w; return {}; }
  mpi::Error WinTest(int w, int* flag) override {
    ++tests;
    win = w;
    if (test_flag < 0) { mpi::Error e; e.code = B200MPI_ERR_ARG; e.msg = "no exposure epoch"; return e; }
    *flag = test_flag;
    return {};
  }
};

int main() {
  // before Init the default implementation reports "not initialised"
  mpi::Window w0;
  bool done = true;
  assert(w0.Post({0, 1}).code == B200MPI_ERR_NOT_INIT && w0.Start({}).code == B200MPI_ERR_NOT_INIT);
  assert(w0.Complete().code == B200MPI_ERR_NOT_INIT && w0.Wait().code == B200MPI_ERR_NOT_INIT);
  assert(w0.Test(&done).code == B200MPI_ERR_NOT_INIT && done);

  Fake fake;
  mpi::Register(&fake);
  mpi::Window w;
  w.id = 17;

  assert(!w.Post({2, 0}) && fake.posts == 1 && fake.count == 2 && fake.group == std::vector<int>({2, 0}) && fake.win == 17);
  assert(!w.Start({1}) && fake.starts == 1 && fake.count == 1 && fake.group == std::vector<int>({1}));
  assert(!w.Post({}) && fake.posts == 2 && fake.count == 0 && fake.group.empty()); // an empty group is legal
  assert(!w.Complete() && fake.completes == 1 && fake.win == 17);
  assert(!w.Wait() && fake.waits == 1);
  assert(!w.Test(&done) && fake.tests == 1 && done);
  fake.test_flag = 0;
  assert(!w.Test(&done) && !done);
  fake.test_flag = -1;
  done = true;
  assert(w.Test(&done).code == B200MPI_ERR_ARG && done && fake.tests == 3); // an error leaves the flag alone

  // an implementation without these calls says so
  Plain plain;
  mpi::mpier() = &plain;
  assert(w.Post({0}).code == B200MPI_ERR_UNSUPPORTED && w.Start({0}).code == B200MPI_ERR_UNSUPPORTED);
  assert(w.Complete().code == B200MPI_ERR_UNSUPPORTED && w.Wait().code == B200MPI_ERR_UNSUPPORTED);
  assert(w.Test(&done).code == B200MPI_ERR_UNSUPPORTED);
  printf("pscw facade ok\n");
  return 0;
}
