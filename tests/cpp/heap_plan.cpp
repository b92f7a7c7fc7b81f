// Replays a sequence of allocations against a host build of the device-heap sub-allocator
// (mpi_b200/csrc/heap.cpp) without any device memory, so that a test can check where a plan of
// buffers lands in a heap of any size.  Commands on stdin, one per line:
//   reset <heap bytes>   an empty heap with the control region (kHeapReserved) in front
//   alloc <bytes>        prints "<offset>" or "nomem"
//   free <offset>        prints "ok" or "error"
//   used                 prints the bytes held by live allocations
#include <cstdio>
#include <cstring>

#include "../../mpi_b200/csrc/heap.h"

int main() {
  b200::Heap h;
  char cmd[32];
  unsigned long long v = 0;
  while (scanf("%31s", cmd) == 1) {
    if (!strcmp(cmd, "used")) {
      printf("%zu\n", h.used());
    } else if (scanf("%llu", &v) != 1) {
      return 2;
    } else if (!strcmp(cmd, "reset")) {
      h.reset_allocator((size_t)v, b200::kHeapReserved, reinterpret_cast<void*>(0x100000000ull));
      printf("ok\n");
    } else if (!strcmp(cmd, "alloc")) {
      size_t off = 0;
      if (h.alloc((size_t)v, off)) printf("nomem\n");
      else printf("%zu\n", off);
    } else if (!strcmp(cmd, "free")) {
      printf(h.free_off((size_t)v) ? "error\n" : "ok\n");
    } else {
      return 2;
    }
    fflush(stdout);
  }
  return 0;
}
