// Host-side check of split16 (kernels.cuh), the split of a ReduceScatterv block into head elements,
// whole 16-byte vectors and tail elements: for every element size, every start residue mod 16 and
// counts 0 ... 3 * EPV + 1 plus a few large ones, every element is covered exactly once, the vectors
// start on a 16-byte boundary, the head stops at the first one and the tail is shorter than a vector.
// Compiled with nvcc, runs on the CPU.
#include <cstdio>
#include <vector>

#include "../../mpi_b200/csrc/kernels.cuh"

static int fail(const char* why, size_t es, uint64_t addr, size_t count) {
  printf("%s (es=%zu addr=%llu count=%zu)\n", why, es, (unsigned long long)addr, count);
  return 1;
}

int main() {
  long checked = 0;
  const size_t large[] = {1000, 4095, 4096, 4097, 65537, 1000003};
  for (size_t es : {1, 2, 4, 8}) {
    const size_t epv = 16 / es;
    std::vector<size_t> counts;
    for (size_t c = 0; c <= 3 * epv + 1; ++c) counts.push_back(c);
    for (size_t c : large) counts.push_back(c);
    for (uint64_t base : {(uint64_t)0, (uint64_t)512, (uint64_t)(1u << 20) + 4096})
      for (uint64_t res = 0; res < 16; ++res)
        for (size_t count : counts) {
          const uint64_t addr = base + res;
          const b200::Split16 s = b200::split16(addr, count, es);
          if (s.head + s.nvec * epv + s.tail != count) return fail("parts do not add up to the block", es, addr, count);
          std::vector<unsigned char> hits(count, 0);
          for (size_t e = 0; e < s.head; ++e) ++hits[e];
          for (size_t i = 0; i < s.nvec; ++i) {
            if ((addr + (s.head + i * epv) * es) % 16) return fail("vector not 16-byte aligned", es, addr, count);
            for (size_t k = 0; k < epv; ++k) ++hits[s.head + i * epv + k];
          }
          for (size_t e = s.head + s.nvec * epv; e < count; ++e) ++hits[e];
          for (size_t e = 0; e < count; ++e)
            if (hits[e] != 1) return fail("element not covered exactly once", es, addr, count);
          if (addr % es) { // misaligned for the type: no boundary on an element edge, all head
            if (s.head != count || s.nvec || s.tail) return fail("misaligned start split into vectors", es, addr, count);
          } else {
            const size_t to_boundary = ((16 - addr % 16) % 16) / es;
            if (count > to_boundary && s.head != to_boundary) return fail("head does not stop at the first boundary", es, addr, count);
            if (count <= to_boundary && (s.head != count || s.nvec || s.tail)) return fail("short block not all head", es, addr, count);
            if (s.tail >= epv) return fail("tail holds a whole vector", es, addr, count);
            if (count >= to_boundary + epv && s.nvec == 0) return fail("room for a vector but none taken", es, addr, count);
          }
          ++checked;
        }
  }
  printf("split16 ok (%ld cases)\n", checked);
  return 0;
}
