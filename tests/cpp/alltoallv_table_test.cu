// CPU checks of the Alltoallv table helper of kernels.cuh (a2av_tables): for worlds of 1 to 8 and
// random and edge matrices of block sizes, the digests of a consistent matrix sum to 0, every
// single-entry change and every swap of two unequal entries in one rank's row or column makes the
// sum nonzero, and the displacements are the prefix sums.  Host code only: no GPU is touched.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../mpi_b200/csrc/kernels.cuh"

using namespace b200;
using Matrix = std::vector<std::vector<size_t>>; // m[src][dst] = elements rank src sends to rank dst

static int failures = 0;
#define CHECK(cond, ...)                         \
  do {                                           \
    if (!(cond)) {                               \
      if (++failures <= 20) {                    \
        printf("FAIL %s:%d: ", __FILE__, __LINE__); \
        printf(__VA_ARGS__);                     \
        printf("\n");                            \
      }                                          \
    }                                            \
  } while (0)

static uint64_t rng_state = 0x2545f4914f6cdd1dull;
static uint64_t next_rand() {
  rng_state += 0x9e3779b97f4a7c15ull;
  return mix64(rng_state);
}

static std::vector<size_t> row_of(const Matrix& m, int i) { return m[i]; }
static std::vector<size_t> col_of(const Matrix& m, int i) {
  std::vector<size_t> c(m.size());
  for (size_t k = 0; k < m.size(); ++k) c[k] = m[k][i];
  return c;
}

static uint64_t digest_of(int me, int n, const std::vector<size_t>& s, const std::vector<size_t>& r, size_t es) {
  VTable sv, rv;
  uint64_t d = 0;
  const bool ok = a2av_tables(me, n, s.data(), r.data(), es, sv, rv, d);
  CHECK(ok, "a2av_tables refused a small table (n=%d)", n);
  return d;
}

// Sum of every rank's digest when rank `who` holds row `s` and column `r` instead of its own.
static uint64_t world_sum(const Matrix& m, size_t es, int who, const std::vector<size_t>& s, const std::vector<size_t>& r) {
  const int n = (int)m.size();
  uint64_t sum = 0;
  for (int i = 0; i < n; ++i) sum += i == who ? digest_of(i, n, s, r, es) : digest_of(i, n, row_of(m, i), col_of(m, i), es);
  return sum;
}

static void check_matrix(const Matrix& m, size_t es, const char* what) {
  const int n = (int)m.size();
  CHECK(world_sum(m, es, -1, {}, {}) == 0, "%s n=%d es=%zu: consistent matrix does not sum to 0", what, n, es);
  for (int i = 0; i < n; ++i) {
    const std::vector<size_t> row = row_of(m, i), col = col_of(m, i);
    // displacements are the prefix sums, in bytes; entries past n hold the total
    VTable sv, rv;
    uint64_t d;
    a2av_tables(i, n, row.data(), col.data(), es, sv, rv, d);
    uint64_t so = 0, ro = 0;
    for (int r = 0; r <= kMaxRanks; ++r) {
      CHECK(sv.off[r] == so && rv.off[r] == ro, "%s n=%d rank %d: displacement %d", what, n, i, r);
      if (r < n) { so += row[r] * es; ro += col[r] * es; }
    }
    // every single-entry change of the row or of the column
    for (int j = 0; j < n; ++j) {
      const size_t deltas[] = {1, 2, 1000, (size_t)1 << 40};
      for (size_t delta : deltas) {
        for (int sign = 0; sign < 2; ++sign) {
          std::vector<size_t> s2 = row, r2 = col;
          if (!sign || row[j] >= delta) {
            s2[j] = sign ? row[j] - delta : row[j] + delta;
            CHECK(world_sum(m, es, i, s2, col) != 0, "%s n=%d: rank %d send_counts[%d] changed by %s%zu unnoticed", what, n, i, j, sign ? "-" : "+", delta);
          }
          if (!sign || col[j] >= delta) {
            r2[j] = sign ? col[j] - delta : col[j] + delta;
            CHECK(world_sum(m, es, i, row, r2) != 0, "%s n=%d: rank %d recv_counts[%d] changed by %s%zu unnoticed", what, n, i, j, sign ? "-" : "+", delta);
          }
        }
      }
      std::vector<size_t> z = row;
      if (row[j] != 0) {
        z[j] = 0;
        CHECK(world_sum(m, es, i, z, col) != 0, "%s n=%d: rank %d send_counts[%d] zeroed unnoticed", what, n, i, j);
      }
    }
    // every swap of two unequal entries in the row or in the column
    for (int j = 0; j < n; ++j)
      for (int k = j + 1; k < n; ++k) {
        if (row[j] != row[k]) {
          std::vector<size_t> s2 = row;
          std::swap(s2[j], s2[k]);
          CHECK(world_sum(m, es, i, s2, col) != 0, "%s n=%d: rank %d send_counts[%d] <-> [%d] unnoticed", what, n, i, j, k);
        }
        if (col[j] != col[k]) {
          std::vector<size_t> r2 = col;
          std::swap(r2[j], r2[k]);
          CHECK(world_sum(m, es, i, row, r2) != 0, "%s n=%d: rank %d recv_counts[%d] <-> [%d] unnoticed", what, n, i, j, k);
        }
      }
  }
}

int main() {
  const size_t sizes[] = {1, 4, 8};
  int matrices = 0;
  for (int n = 1; n <= kMaxRanks; ++n) {
    for (size_t es : sizes) {
      Matrix zeros(n, std::vector<size_t>(n, 0)), diag = zeros, one = zeros;
      for (int i = 0; i < n; ++i) diag[i][i] = 17 + i;
      one[n - 1][0] = (size_t)1 << 24;
      check_matrix(zeros, es, "zeros");
      check_matrix(diag, es, "diagonal");
      check_matrix(one, es, "one pair");
      matrices += 3;
      const size_t pick[] = {0, 1, 3, 5, 257, 4099, 65537};
      for (int trial = 0; trial < 6; ++trial) {
        Matrix m = zeros;
        for (int i = 0; i < n; ++i)
          for (int j = 0; j < n; ++j) m[i][j] = trial % 2 ? pick[next_rand() % 7] : next_rand() % 100000;
        check_matrix(m, es, "random");
        ++matrices;
      }
    }
  }
  // a count whose byte size, or a sum of byte sizes, does not fit in 64 bits is refused
  {
    VTable sv, rv;
    uint64_t d;
    const size_t big[2] = {(size_t)1 << 62, 0}, two[2] = {(size_t)1 << 62, (size_t)1 << 62}, zero[2] = {0, 0};
    CHECK(!a2av_tables(0, 2, big, zero, 8, sv, rv, d), "count * 8 overflow accepted");
    CHECK(!a2av_tables(0, 2, zero, two, 4, sv, rv, d), "sum overflow accepted");
    CHECK(a2av_tables(0, 2, two, zero, 1, sv, rv, d), "a sum that fits was refused");
  }
  if (failures) {
    printf("%d failures\n", failures);
    return 1;
  }
  printf("alltoallv table ok (%d matrices)\n", matrices);
  return 0;
}
