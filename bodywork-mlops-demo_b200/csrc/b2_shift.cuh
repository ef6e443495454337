// b2_shift.cuh -- undo the per-column shift: S = [X 1 y]^T [X 1 y] from the moments of the shifted rows.
//
// The tensor-core and narrow Gram paths accumulate moments of v = x - c and y' = y - c_y (c from gram_shift.cu); their
// folds supply those moments and this header turns them into the entries of S in fp64.  The algebra is exact for every
// c.  Index space of S (stride d + 2): features 0..d-1, d = ones, d + 1 = y.
#pragma once

#include "b2_internal.cuh"

namespace b2 {

// Entry (a, b), a <= b, of S; evaluate (b, a) with the same (a, b), so that S is exactly symmetric.  c[j]: the shift of
// feature j, c[kMaxD]: the shift of y.  The moments of the shifted rows:
//   G(i, j) = sum v_i v_j, s1(i) = sum v_i, sxy(i) = sum v_i y', n = rows used, sy = sum y', syy = sum y'^2.
template <typename CT, typename FG, typename FS1, typename FSXY>
__device__ __forceinline__ double unshift_entry(int a, int b, int d, const CT* c, FG G, FS1 s1, FSXY sxy, double n,
                                                double sy, double syy) {
  const double cy = (double)c[kMaxD];
  if (b < d) {
    const double ca = (double)c[a], cb = (double)c[b];
    return G(a, b) + ca * s1(b) + cb * s1(a) + n * ca * cb;
  }
  if (a < d) {
    const double ci = (double)c[a];
    if (b == d) return s1(a) + n * ci;
    return sxy(a) + cy * s1(a) + ci * sy + n * ci * cy;
  }
  if (a == d && b == d) return n;
  if (a == d + 1) return syy + 2.0 * cy * sy + n * cy * cy;
  return sy + n * cy;
}

}  // namespace b2
