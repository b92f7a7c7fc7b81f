// Host-side run of the device ops of MAXLOC / MINLOC (OpMaxLoc, OpMinLoc in kernels.cuh) on the same
// inputs as the numpy restatement.  Usage: loc_op_test <dtype 1|2|3> <op 1|2> <n> <count> <in> <out>
// where <in> holds n ranks of count 16-byte pairs, rank after rank.  The pairs of every element are
// folded with Op::apply in rank order from the left, from the right and as a pairwise tree; the
// three must agree byte for byte, and the left fold is written to <out>.  Compiled with nvcc, runs
// on the CPU.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../mpi_b200/csrc/kernels.cuh"

template <typename V, typename Op>
static int run(int n, size_t count, const std::vector<b200::Loc<V>>& in, std::vector<b200::Loc<V>>& out) {
  using P = b200::Loc<V>;
  for (size_t e = 0; e < count; ++e) {
    P x[b200::kMaxRanks];
    for (int r = 0; r < n; ++r) x[r] = in[(size_t)r * count + e];
    P left = x[0];
    for (int r = 1; r < n; ++r) left = Op::template apply<P>(left, x[r]);
    P right = x[n - 1];
    for (int r = n - 2; r >= 0; --r) right = Op::template apply<P>(x[r], right);
    P t[b200::kMaxRanks];
    int m = n;
    for (int r = 0; r < n; ++r) t[r] = x[r];
    while (m > 1) { // neighbours level by level, lower ranks on the left
      int k = 0;
      for (int r = 0; r + 1 < m; r += 2) t[k++] = Op::template apply<P>(t[r], t[r + 1]);
      if (m % 2) t[k++] = t[m - 1];
      m = k;
    }
    if (memcmp(&left, &right, sizeof(P)) || memcmp(&left, &t[0], sizeof(P))) {
      printf("bracketings differ at element %zu\n", e);
      return 1;
    }
    out[e] = left;
  }
  return 0;
}

template <typename V>
static int by_op(int op, int n, size_t count, FILE* fi, FILE* fo) {
  std::vector<b200::Loc<V>> in((size_t)n * count), out(count);
  if (fread(in.data(), 16, in.size(), fi) != in.size()) return printf("short input\n"), 1;
  const int rc = op == 1 ? run<V, b200::OpMaxLoc>(n, count, in, out) : run<V, b200::OpMinLoc>(n, count, in, out);
  if (rc) return rc;
  if (fwrite(out.data(), 16, count, fo) != count) return printf("short output\n"), 1;
  return 0;
}

int main(int argc, char** argv) {
  if (argc != 7) return printf("usage: loc_op_test dtype op n count in out\n"), 2;
  const int dtype = atoi(argv[1]), op = atoi(argv[2]), n = atoi(argv[3]);
  const size_t count = strtoull(argv[4], nullptr, 10);
  if (n < 1 || n > b200::kMaxRanks || (op != 1 && op != 2)) return printf("bad arguments\n"), 2;
  FILE* fi = fopen(argv[5], "rb");
  FILE* fo = fopen(argv[6], "wb");
  if (!fi || !fo) return printf("cannot open files\n"), 2;
  int rc = 2;
  if (dtype == 1) rc = by_op<long long>(op, n, count, fi, fo);
  else if (dtype == 2) rc = by_op<float>(op, n, count, fi, fo);
  else if (dtype == 3) rc = by_op<double>(op, n, count, fi, fo);
  fclose(fi);
  fclose(fo);
  if (rc == 0) printf("loc op ok\n");
  return rc;
}
