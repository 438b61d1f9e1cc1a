// group_block.cuh -- one block of the grouped block-Jacobi preconditioner of gmres.cu: gather J[R_g, C_g] from a CSR
// matrix and invert it by Gauss-Jordan with partial pivoting.  A group g is a list of rows R_g and a list of columns C_g
// of equal size s <= 32 (one matrix cell, or one fracture cell with its two mortar cells, of the fractured contact models:
// their complementarity rows have zero diagonals, so the pivoting is required).
//
// The routines work on one row (gather, elimination) or one column (row swap) of the s x s row-major block A and of the
// inverse E: the device runs one warp per group with lane i on row / column i, the host build in tests/emu runs the
// same routines in a loop.  Within one elimination step every row update reads only its own row and the pivot row, and
// the pivot row is scaled after all other rows are updated, so the loop order does not change the result.
#pragma once
#include <cmath>
#include <cstdint>

#include "views.hpp"

namespace pb {

constexpr int kGroupMax = 32;

// row i of the block: a_row[j] = sum of the entries of CSR row `row` in column cols[j]; entries outside C_g are ignored
PB_HD void group_gather_row(const int32_t *ip, const int32_t *ix, const double *data, int64_t row, const int32_t *cols,
                            int s, double *a_row) {
    for (int j = 0; j < s; ++j) a_row[j] = 0.0;
    for (int32_t q = ip[row]; q < ip[row + 1]; ++q) {
        const int32_t c = ix[q];
        for (int j = 0; j < s; ++j)
            if (cols[j] == c) { a_row[j] += data[q]; break; }
    }
}

// pivot of step k: the row p >= k with the largest |A[p][k]| (the first one on ties); -1 if that is zero or not finite
PB_HD int group_pivot(const double *A, int s, int k) {
    int p = k;
    double best = fabs(A[k * s + k]);
    for (int i = k + 1; i < s; ++i) {
        const double v = fabs(A[i * s + k]);
        if (v > best) { best = v; p = i; }
    }
    return (best > 0.0 && best <= 1.79769313486231570e308) ? p : -1;
}

// column l of the swap of rows k and p, in A and in E
PB_HD void group_swap_col(double *A, double *E, int s, int k, int p, int l) {
    if (p == k) return;
    double t = A[k * s + l]; A[k * s + l] = A[p * s + l]; A[p * s + l] = t;
    t = E[k * s + l]; E[k * s + l] = E[p * s + l]; E[p * s + l] = t;
}

// row i != k: row_i -= (A[i][k] / A[k][k]) row_k, in A and in E
PB_HD void group_eliminate_row(double *A, double *E, int s, int k, int i) {
    const double f = A[i * s + k] / A[k * s + k];
    if (f == 0.0) return;
    for (int j = 0; j < s; ++j) {
        A[i * s + j] -= f * A[k * s + j];
        E[i * s + j] -= f * E[k * s + j];
    }
}

// the pivot row, after every other row of step k: row_k /= A[k][k]
PB_HD void group_scale_row(double *A, double *E, int s, int k) {
    const double inv = 1.0 / A[k * s + k];
    for (int j = 0; j < s; ++j) {
        A[k * s + j] *= inv;
        E[k * s + j] *= inv;
    }
}

// E = I (row i)
PB_HD void group_identity_row(double *E, int s, int i) {
    for (int j = 0; j < s; ++j) E[i * s + j] = i == j ? 1.0 : 0.0;
}

// The whole inversion, serially (the host build): A is destroyed, E receives A^-1.  Returns the failing step or -1.
PB_HD int group_invert_serial(double *A, double *E, int s) {
    for (int i = 0; i < s; ++i) group_identity_row(E, s, i);
    for (int k = 0; k < s; ++k) {
        const int p = group_pivot(A, s, k);
        if (p < 0) return k;
        for (int l = 0; l < s; ++l) group_swap_col(A, E, s, k, p, l);
        for (int i = 0; i < s; ++i)
            if (i != k) group_eliminate_row(A, E, s, k, i);
        group_scale_row(A, E, s, k);
    }
    return -1;
}

}  // namespace pb
