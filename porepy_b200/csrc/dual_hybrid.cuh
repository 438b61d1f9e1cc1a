// dual_hybrid.cuh -- hybridization of the mixed schemes MVEM and RT0: each cell's local saddle system
//   [A B C; B^T 0 0] [v; p; lambda] = [r; h; -],   B = -1 (n x 1), C = I,
// with v the cell's outward face fluxes and lambda one pressure per face, is condensed exactly onto lambda
// (reference numerics/vem/hybrid.py, HybridDualVEM.matrix_rhs):
//   E = A^-1,  z = E B,  t = B^T E B,  S = 1 / t,  L = z S z^T - E,
//   p = S (z^T r - z^T lambda - h),  v = E (r - B p - lambda) = E r - z p - E lambda,
// so that the continuity rows sum_cells v = q become sum_cells L lambda = q + sum_cells (L r - S z h).
// HybridDualVEM writes its source f as h = -f and no r (hybrid.py: rhs += z S f, p = S (f - z^T lambda)).
//
// The routines work on one lane = one local face i of one cell: row i of A (dual_cell.cuh's row routine with the
// DualLocalRow sink), the Gauss-Jordan inverse of group_block.cuh, then row i of L and the rhs term.  The device runs
// one warp per cell with the per-cell arrays in shared memory (dual.cu); the test-only host build in tests/emu loops
// over the lanes.  Within one step every lane reads only what the previous step finished, so the loop order does not
// change the result.
#pragma once
#include <cmath>
#include <cstdint>

#include "../../include/poreb200.h"
#include "dual_cell.cuh"
#include "group_block.cuh"

namespace pb {

constexpr int kHybridMaxFaces = 32;   // one lane per face

// Per-cell work arrays: A and E (n x n row-major), z, r and lambda (n each).
PB_HD int hybrid_cell_doubles(int n) { return 2 * n * n + 3 * n; }

// What the two uses read besides the discretization's topology and geometry.
//   mode PB_DUAL_HYBRID_VEM:    values = [bc_values (nf); source (nc)], aperture per cell; r = 0, h = -source.
//   mode PB_DUAL_HYBRID_SADDLE: values = b of the saddle-point system (nf + nc), codes PB_BC_* per face; lambda = 0 on
//     the fixed faces (hybrid_fixed); r_i = s_i b_f on the faces whose first cell this is, except Neumann faces.
struct HybridIn {
    int mode;
    int64_t nf;
    const int32_t *fc_ip, *fc_cell;   // the cells of every face, ascending
    const double *aperture;           // VEM mode; NULL elsewhere
    const double *values;
    const uint8_t *codes;             // saddle mode
};

// A face whose pressure is given: Dirichlet, or a boundary face without a condition, which the saddle-point system
// also treats as a pressure condition (its row keeps the mass row and the divergence column).
PB_HD bool hybrid_fixed(const HybridIn &H, int32_t f) {
    const uint8_t code = H.codes[f];
    return code == PB_BC_DIR || (code == PB_BC_INTERIOR && H.fc_ip[f + 1] - H.fc_ip[f] == 1);
}

// Sign of face f in its first cell (the orientation of the saddle-point system's face unknown).
PB_HD double hybrid_face_sign(const DualTopo &T, const HybridIn &H, int32_t f) {
    const int32_t c = H.fc_cell[H.fc_ip[f]];
    int32_t lo = T.cf_ip[c], hi = T.cf_ip[c + 1];
    while (lo < hi) {
        const int32_t mid = (lo + hi) >> 1;
        if (T.cf_ix[mid] < f) lo = mid + 1; else hi = mid;
    }
    return (double)T.cf_sg[lo];
}

// Lane i: row i of the cell's local matrix in outward-flux variables into A (n x n).
template <int ND>
PB_HD void hybrid_local_row(int method, int64_t c, int i, const DualTopo &T, const DualGeo &G, const HybridIn &H,
                            double *A, int32_t *bad) {
    const int b = T.cf_ip[c], n = T.cf_ip[c + 1] - b;
    const DualLocalRow out{A + i * n, (double)T.cf_sg[b + i], H.aperture ? 1.0 / H.aperture[c] : 1.0, b};
    if (method == kDualMvem) mvem_row<ND>(b + i, T, G, out, bad);
    else rt0_row<ND>(b + i, T, G, out);
}

// Lane i, after the inversion (E = A^-1): z_i = (E B)_i, r_i and lambda_i (lam may be NULL: the condensation).
PB_HD void hybrid_vectors(int64_t c, int i, const DualTopo &T, const HybridIn &H, const double *E, const double *lam,
                          double *z, double *r, double *lv) {
    const int b = T.cf_ip[c], n = T.cf_ip[c + 1] - b;
    const int32_t f = T.cf_ix[b + i];
    double s = 0.0;
    for (int j = 0; j < n; ++j) s += E[i * n + j];
    z[i] = -s;
    double ri = 0.0, li = lam ? lam[f] : 0.0;
    if (H.mode == PB_DUAL_HYBRID_SADDLE) {
        if (H.fc_cell[H.fc_ip[f]] == (int32_t)c && H.codes[f] != PB_BC_NEU) ri = (double)T.cf_sg[b + i] * H.values[f];
        if (hybrid_fixed(H, f)) li = 0.0;
    }
    r[i] = ri;
    lv[i] = li;
}

// h of the cell and t = B^T E B = -sum z (every lane sums in the same order)
PB_HD double hybrid_h(int64_t c, const HybridIn &H) {
    return H.mode == PB_DUAL_HYBRID_VEM ? -H.values[H.nf + c] : H.values[H.nf + c];
}

PB_HD double hybrid_t(const double *z, int n) {
    double t = 0.0;
    for (int j = 0; j < n; ++j) t -= z[j];
    return t;
}

// Lane i of the condensation: row i of L added into the face matrix (values in the mass pattern), and
// (L r)_i - S z_i h added into the face right-hand side.  At most two cells add to one entry, into zeroed values.
PB_HD void hybrid_condense_row(int64_t c, int i, const DualTopo &T, const HybridIn &H, const double *E, const double *z,
                               const double *r, double *hval, double *rhs) {
    const int b = T.cf_ip[c], n = T.cf_ip[c + 1] - b;
    const double S = 1.0 / hybrid_t(z, n);
    const int32_t fi = T.cf_ix[b + i];
    double acc = 0.0;
    for (int j = 0; j < n; ++j) {
        const double l = z[i] * S * z[j] - E[i * n + j];
        dual_add(hval + dual_pos(T, fi, T.cf_ix[b + j]), l);
        acc += l * r[j];
    }
    dual_add(rhs + fi, acc - S * z[i] * hybrid_h(c, H));
}

// Lane i of the recovery: p = S (z^T r - z^T lambda - h) (lane 0 writes it) and u_f = s_i v_i, v = E (r - B p - lambda),
// written by the face's first cell only.
PB_HD void hybrid_recover_row(int64_t c, int i, const DualTopo &T, const HybridIn &H, const double *E, const double *z,
                              const double *r, const double *lv, double *u, double *p) {
    const int b = T.cf_ip[c], n = T.cf_ip[c + 1] - b;
    double zr = 0.0, zl = 0.0;
    for (int j = 0; j < n; ++j) {
        zr += z[j] * r[j];
        zl += z[j] * lv[j];
    }
    const double pc = (zr - zl - hybrid_h(c, H)) / hybrid_t(z, n);
    if (i == 0) p[c] = pc;
    const int32_t fi = T.cf_ix[b + i];
    if (H.fc_cell[H.fc_ip[fi]] != (int32_t)c) return;
    double v = 0.0;
    for (int j = 0; j < n; ++j) v += E[i * n + j] * (r[j] + pc - lv[j]);
    u[fi] = (double)T.cf_sg[b + i] * v;
}

// Row f of the face system after the condensation.  norm: |H|_inf before the boundary conditions (VEM mode) or
// |mass|_inf of the saddle-point system (saddle mode).
//   VEM mode (hybrid.py): Dirichlet rows cleared with norm on the diagonal and rhs norm bc; Neumann rhs += s bc area.
//   Saddle mode: fixed faces get identity rows and zeroed columns (lambda = 0, their data is already in r); Robin
//   faces add -robin_weight area on the diagonal (lambda = v / (robin_weight area) there); Neumann faces add
//   s b_f / norm, the flux their saddle-point row prescribes.
PB_HD void hybrid_bc_row(int32_t f, const DualTopo &T, const HybridIn &H, const double *robin_weight,
                         const double *face_areas, double norm, double *hval, double *rhs) {
    const uint8_t code = H.codes[f];
    const int32_t q0 = T.mass_ip[f], q1 = T.mass_ip[f + 1];
    if (H.mode == PB_DUAL_HYBRID_VEM) {
        if (code == PB_BC_DIR) {
            for (int32_t q = q0; q < q1; ++q) hval[q] = T.mass_ix[q] == f ? norm : 0.0;
            rhs[f] = norm * H.values[f];
        } else if (code == PB_BC_NEU) {
            rhs[f] += hybrid_face_sign(T, H, f) * H.values[f] * face_areas[f];
        }
        return;
    }
    if (hybrid_fixed(H, f)) {
        for (int32_t q = q0; q < q1; ++q) hval[q] = T.mass_ix[q] == f ? 1.0 : 0.0;
        rhs[f] = 0.0;
        return;
    }
    for (int32_t q = q0; q < q1; ++q) {
        if (hybrid_fixed(H, T.mass_ix[q])) hval[q] = 0.0;
        else if (T.mass_ix[q] == f && code == PB_BC_ROB) hval[q] -= robin_weight[f] * face_areas[f];
    }
    if (code == PB_BC_NEU) rhs[f] += hybrid_face_sign(T, H, f) * H.values[f] / norm;
}

}  // namespace pb
