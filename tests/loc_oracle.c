/*
 * tests/loc_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Compiled on first use by
 * tests/_loc_oracle.py; libb200mpi never calls it.
 *
 * CPU restatement of MAXLOC / MINLOC (b200mpi_allreduce_loc, b200mpi_reduce_loc).  An element is
 * the 16-byte pair { V val; int64_t loc; } with V = i64 (dtype 1), f32 (2) or f64 (3); an f32 value
 * is followed by 4 padding bytes.  op 1 is MAXLOC, 2 MINLOC.  The pairs of ranks 0..n-1 are folded
 * in rank order: acc = x_0, then x_r replaces acc exactly when
 *   - x_r.val is better than acc.val (greater for MAXLOC, smaller for MINLOC), or
 *   - the two values are equal and x_r.loc < acc.loc (signed).
 * i64 values use the signed order.  Floats compare as IEEE (-0 == +0), except that every NaN is
 * better than every number under both ops and all NaNs are equal.  The winning pair is copied
 * whole (value bits, loc and padding).  Among the pairs with the best (value, loc), the lowest
 * rank's is the result, whatever the bracketing.
 */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

/* 1: b replaces a (a holds the lower ranks) */
static int replaces(int dtype, int op, const unsigned char* a, const unsigned char* b) {
  int64_t la, lb;
  int better, equal;
  memcpy(&la, a + 8, 8);
  memcpy(&lb, b + 8, 8);
  if (dtype == 1) {
    int64_t x, y;
    memcpy(&x, a, 8);
    memcpy(&y, b, 8);
    better = op == 1 ? y > x : y < x;
    equal = x == y;
  } else {
    double x, y; /* f32 widens exactly: the order, -0 == +0 and NaN-ness are kept */
    if (dtype == 2) {
      float fx, fy;
      memcpy(&fx, a, 4);
      memcpy(&fy, b, 4);
      x = fx;
      y = fy;
    } else {
      memcpy(&x, a, 8);
      memcpy(&y, b, 8);
    }
    const int xnan = x != x, ynan = y != y;
    if (xnan || ynan) {
      better = !xnan && ynan;
      equal = xnan && ynan;
    } else {
      better = op == 1 ? y > x : y < x;
      equal = x == y;
    }
  }
  return better || (equal && lb < la);
}

/* in[r] holds rank r's `count` pairs; out receives the `count` winning pairs */
int oracle_allreduce_loc(int dtype, int op, int n, size_t count, const void* const* in, void* out) {
  if (n < 1 || n > 8 || dtype < 1 || dtype > 3 || (op != 1 && op != 2)) return -1;
  for (size_t e = 0; e < count; ++e) {
    unsigned char acc[16];
    memcpy(acc, (const unsigned char*)in[0] + 16 * e, 16);
    for (int r = 1; r < n; ++r) {
      const unsigned char* b = (const unsigned char*)in[r] + 16 * e;
      if (replaces(dtype, op, acc, b)) memcpy(acc, b, 16);
    }
    memcpy((unsigned char*)out + 16 * e, acc, 16);
  }
  return 0;
}
