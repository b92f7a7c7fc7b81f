/*
 * tests/gather_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Compiled on first use by
 * tests/_gather_oracle.py; libb200mpi never calls it.
 *
 * CPU restatement of what a value means after the rooted and variable-count collectives:
 *
 *   Gatherv   root's recv == send_0 ++ send_1 ++ ... ++ send_{n-1}, send_r holding counts[r]
 *             elements (displacement of r = counts[0] + ... + counts[r-1]); Allgatherv: the same
 *             on every rank; Gather: the uniform table (== Allgather on root).
 *   Scatterv  rank me's recv == root's send[displ[me] .. displ[me] + counts[me]); Scatter: the
 *             uniform table.  Scatter(Gather(x)) == x.
 * Nothing is reduced, so every result is bit-exact for every element type.
 */
#include <stddef.h>
#include <string.h>

/* in[r] holds counts[r] elements of `esize` bytes; out (their sum) is root's recv */
int oracle_gatherv(size_t esize, int n, const size_t* counts, const void* const* in, void* out) {
  size_t off = 0;
  if (n < 1 || n > 8) return -1;
  for (int r = 0; r < n; ++r) {
    const size_t b = counts[r] * esize;
    if (b) memcpy((char*)out + off, in[r], b);
    off += b;
  }
  return 0;
}

/* root_send holds sum(counts) elements; out (counts[me] elements) is what rank `me` receives */
int oracle_scatterv(size_t esize, int n, int me, const size_t* counts, const void* root_send, void* out) {
  size_t off = 0;
  if (n < 1 || n > 8 || me < 0 || me >= n) return -1;
  for (int r = 0; r < me; ++r) off += counts[r] * esize;
  if (counts[me]) memcpy(out, (const char*)root_send + off, counts[me] * esize);
  return 0;
}
