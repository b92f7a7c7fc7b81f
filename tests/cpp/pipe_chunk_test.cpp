// Host-side check of pipe_chunk_elems (hostutil.h), the chunk size of the pipelined host-slice
// Allreduce, Bcast and Allgather.  Compiled with g++, runs on the CPU.
//
// Without arguments: over element sizes, rows, world sizes and knob pairs, the chunk is a multiple of
// 4096 elements and at least 4096; in a world of more than one rank it does not depend on whether
// this rank bounces its buffer; a bouncing rank and a world of one keep the rule the library had
// before (restated here as old_chunk_elems), so only pinned and registered ranks of a multi-rank
// world see a new schedule.  Prints "pipe_chunk ok".
//
// With arguments  pipe_chunk_bytes bounce_chunk_bytes  then groups of  es rows n count : one line per
// group, "chunks old bounce=<a> old direct=<b> new bounce=<c> new direct=<d>", the number of chunk
// launches a rank issues for `count` elements under each rule, bouncing or not.
#include <cstdio>
#include <cstdlib>

#include "../../mpi_b200/csrc/hostutil.h"

using b200::pipe_chunk_elems;

// The rule of the previous release: the bounce chunk caps only the ranks that bounce.
static size_t old_chunk_elems(size_t es, size_t rows, bool bounce, size_t pipe, size_t bnc) {
  size_t bytes = pipe;
  if (bounce) bytes = std::min(bytes, bnc);
  return std::max<size_t>(bytes / rows / es, 4096) / 4096 * 4096;
}

static size_t chunks(size_t count, size_t elems) { return (count + elems - 1) / elems; }

static int fail(const char* why, size_t es, size_t rows, int n, size_t pipe, size_t bnc) {
  printf("FAIL: %s (es=%zu rows=%zu n=%d pipe=%zu bounce=%zu)\n", why, es, rows, n, pipe, bnc);
  return 1;
}

int main(int argc, char** argv) {
  if (argc > 1) {
    if (argc < 3 || (argc - 3) % 4) {
      printf("usage: %s pipe_chunk_bytes bounce_chunk_bytes [es rows n count]...\n", argv[0]);
      return 2;
    }
    const size_t pipe = strtoull(argv[1], nullptr, 0), bnc = strtoull(argv[2], nullptr, 0);
    for (int i = 3; i < argc; i += 4) {
      const size_t es = strtoull(argv[i], nullptr, 0), rows = strtoull(argv[i + 1], nullptr, 0);
      const int n = atoi(argv[i + 2]);
      const size_t count = strtoull(argv[i + 3], nullptr, 0);
      printf("chunks old bounce=%zu old direct=%zu new bounce=%zu new direct=%zu\n",
             chunks(count, old_chunk_elems(es, rows, true, pipe, bnc)), chunks(count, old_chunk_elems(es, rows, false, pipe, bnc)),
             chunks(count, pipe_chunk_elems(es, rows, n, true, pipe, bnc)), chunks(count, pipe_chunk_elems(es, rows, n, false, pipe, bnc)));
    }
    return 0;
  }
  const size_t K = 1024, M = 1024 * 1024;
  const size_t knobs[][2] = {{16 * M, 4 * M}, {4 * M, 16 * M}, {M, 256 * K}, {64 * K, 64 * K}, {64 * K, M}, {100 * K + 3, 64 * K}};
  long checked = 0;
  for (const auto& kb : knobs)
    for (size_t es : {1, 4, 8})
      for (int n = 1; n <= 8; ++n)
        for (size_t rows : {(size_t)1, (size_t)n}) {
          const size_t pipe = kb[0], bnc = kb[1];
          const size_t nb = pipe_chunk_elems(es, rows, n, true, pipe, bnc), nd = pipe_chunk_elems(es, rows, n, false, pipe, bnc);
          for (size_t e : {nb, nd})
            if (e < 4096 || e % 4096) return fail("chunk not a positive multiple of 4096 elements", es, rows, n, pipe, bnc);
          if (nb != old_chunk_elems(es, rows, true, pipe, bnc)) return fail("a bouncing rank's chunk changed", es, rows, n, pipe, bnc);
          if (n == 1 && nd != old_chunk_elems(es, rows, false, pipe, bnc)) return fail("a world of one changed its pinned chunk", es, rows, n, pipe, bnc);
          if (n > 1 && nb != nd) return fail("ranks of one world chunk differently", es, rows, n, pipe, bnc);
          ++checked;
        }
  printf("pipe_chunk ok (%ld cases)\n", checked);
  return 0;
}
