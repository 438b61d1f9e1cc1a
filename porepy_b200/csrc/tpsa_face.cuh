// tpsa_face.cuh -- per-face routine of the two-point stress approximation (Nordbotten & Keilegavlen,
// arXiv:2405.10390; reference numerics/fv/tpsa.py:376-997 with the helpers _create_filters :1000,
// _create_cell_to_face_maps :1070, _compute_distances :1184, _vector_laplace_matrices :1314 and
// _create_numbering :1396).  Every row of the 14 TPSA matrices belongs to one face and every column is one of
// the face's cells (or the face itself for the bound_* terms), so one call writes all values of one face with
// no atomics.  The CUDA kernel (face.cu) runs one thread per face; the test-only host build loops over faces.
#pragma once
#include <cmath>
#include <cstddef>

#include "views.hpp"

namespace pb {

// PB_TPSA_* term indices and block shapes: include/poreb200.h.  o.t[k] == nullptr: term k not wanted.
struct TpsaOut {
    double *t[14];
};

// Length of o.t[k] on a grid of nf faces and nfc (face, cell) entries: the values per entry of the cell terms
// (k < PB_TPSA_BOUND_STRESS = 10) or per face of the bound_* face terms, in the layout below.
constexpr size_t tpsa_term_size(int k, int nd, size_t nfc, size_t nf) {
    const size_t d = nd, r = nd == 3 ? 3 : 1;
    const size_t per[14] = {d, d * r, d, r * d, r * r, d, 1, d, d * r, d, d, r * d, d, d};
    return per[k] * (k < 10 ? nfc : nf);
}

// Value layout, with L = number of cells of face f (1 or 2) and p0 = fc_ptr[f]:
//  * cell terms with br x bc blocks: the CSR order of the expanded pattern (fv.block_expand), i.e. block
//    entry (i, j) of the cell of rank r (ascending cell index) at br*bc*p0 + i*bc*L + r*bc + j.  kron(., I_nd)
//    terms store their nd diagonal values as an nd x 1 block (column c*nd + i of row f*nd + i).
//  * face terms: br x bc row-major at f*br*bc (kron(., I_nd) terms: nd values at f*nd).
// codes / robw: per (face, component) at f*nd + i (BoundaryConditionVectorial flags raveled in "F" order).
// flags[f] != 0: face in sd.get_all_boundary_faces() (it then has exactly one cell, checked by the caller).
template <int ND>
PB_HD void tpsa_face(int64_t f, const GeoView &G, const double *mu, const uint8_t *codes, const double *robw,
                     const uint8_t *flags, const int32_t *face_cells, const int32_t *fc_ptr, const TpsaOut &o) {
    double n[3], xf[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        n[i] = G.fnorm[i * G.face_cs + f * G.face_es];
        xf[i] = G.fcent[i * G.face_cs + f * G.face_es];
    }
    const double A = G.farea[f];

    // the face's cells: index, sign of cell_faces, mu / distance (tpsa.py:1214-1231)
    int64_t cell[2] = {0, 0};
    double sg[2] = {0.0, 0.0}, m[2] = {0.0, 0.0};
    int ncell = 0;
#pragma unroll
    for (int sd = 0; sd < 2; ++sd) {
        const int32_t enc = face_cells[2 * f + sd];
        if (enc < 0) continue;
        const int64_t c = enc >> 1;
        const double s = (enc & 1) ? -1.0 : 1.0;
        double dsum = 0.0;   // all three rows of the normal (:1221-1228)
#pragma unroll
        for (int i = 0; i < 3; ++i) dsum += (n[i] * s) * (xf[i] - G.ccent[i * G.cell_cs + c * G.cell_es]) / A;
        const double mk = mu[c] / fabs(dsum);
        if (ncell == 0) { cell[0] = c; sg[0] = s; m[0] = mk; }
        else { cell[1] = c; sg[1] = s; m[1] = mk; }
        ++ncell;
    }
    if (ncell == 0) return;
    const int L = ncell;
    // rank of slot k in the row (ascending cell index)
    const int rk0 = (ncell == 2 && cell[0] > cell[1]) ? 1 : 0;
    const int rk[2] = {rk0, 1 - rk0};

    double two_m = 0.0, inv_m = 0.0, ssum = 0.0;
#pragma unroll
    for (int k = 0; k < 2; ++k)
        if (k < ncell) { two_m += 2.0 * m[k]; inv_m += 1.0 / m[k]; ssum += sg[k]; }

    double dir[ND], neu[ND], rob[ND], w[ND];
#pragma unroll
    for (int i = 0; i < ND; ++i) {
        const int code = codes[f * ND + i];
        dir[i] = code == 1 ? 1.0 : 0.0;
        neu[i] = code == 2 ? 1.0 : 0.0;
        rob[i] = code == 3 ? 1.0 : 0.0;
        w[i] = (code == 3 && robw) ? robw[f * ND + i] : 0.0;
    }

    // arithmetic_average_shear_modulus (:1251-1260): Robin faces add the weights projected on the unit normal
    double ar_avg = two_m;
    if (rob[0] != 0.0) {
        double proj = 0.0;
#pragma unroll
        for (int i = 0; i < ND; ++i) { const double u = n[i] / A; proj += w[i] * (u * u); }
        ar_avg += proj;
    }
    // scalar Dirichlet filter of solid_mass_total_pressure (:1053-1057): the component of the largest |n| over
    // all three rows, first index on ties
    int imax = 0;
    double amax = fabs(n[0]);
#pragma unroll
    for (int i = 1; i < 3; ++i)
        if (fabs(n[i]) > amax) { amax = fabs(n[i]); imax = i; }
    double dir_np = 1.0;
#pragma unroll
    for (int i = 0; i < ND; ++i)
        if (i == imax && dir[i] != 0.0) dir_np = 0.0;

    double invS[ND], trm[ND], trm_bnd[ND], b2f[ND], pass[ND];
#pragma unroll
    for (int i = 0; i < ND; ++i) {
        const double S = two_m + (rob[i] != 0.0 ? w[i] : 0.0);                    // :1281-1284
        invS[i] = 1.0 / S;
        const double t = 2.0 * A / (inv_m + (rob[i] != 0.0 ? 1.0 / w[i] : 0.0));  // :648-663
        b2f[i] = rob[i] * invS[i] * w[i];                                          // :1141-1147
        trm_bnd[i] = dir[i] != 0.0 ? t : (neu[i] != 0.0 ? 1.0 : (rob[i] != 0.0 ? (1.0 - b2f[i]) + t : 0.0));
        trm[i] = neu[i] != 0.0 ? 0.0 : t;                                          // :1355-1371
        pass[i] = (neu[i] != 0.0 || rob[i] != 0.0) ? 1.0 : 0.0;                   // neu_rob_pass_nd
    }
    const double invA = 1.0 / A;
    const double sA = (flags[f] ? sg[0] : 0.0) / A;                               // sgn_bf / face_areas (:915)

    // rotation operators: 3-D R = [[0,-n2,n1],[n2,0,-n0],[-n1,n0,0]] (:762-767); 2-D v = [n1, -n0] (:800)
    double R[3][3] = {}, RR[3][3] = {}, v[2] = {0.0, 0.0};
    if constexpr (ND == 3) {
        R[0][0] = 0.0;   R[0][1] = -n[2]; R[0][2] = n[1];
        R[1][0] = n[2];  R[1][1] = 0.0;   R[1][2] = -n[0];
        R[2][0] = -n[1]; R[2][1] = n[0];  R[2][2] = 0.0;
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) RR[i][j] = R[i][0] * R[0][j] + R[i][1] * R[1][j] + R[i][2] * R[2][j];
    } else {
        v[0] = n[1]; v[1] = -n[0];
    }
    const double d_rr = 1.0 / (ar_avg * A);
    const int64_t p0 = fc_ptr[f];
    auto at = [&](int br, int bc, int i, int r, int j) -> int64_t {
        return (int64_t)br * bc * p0 + (int64_t)i * bc * L + (int64_t)r * bc + j;
    };

#pragma unroll
    for (int k = 0; k < 2; ++k) {
        if (k >= ncell) break;
        const int r = rk[k];
        const double s = sg[k];
        double c2f[ND];   // c2f and c2f_scalar_2_nd: zero on Dirichlet components (:1116-1162)
#pragma unroll
        for (int i = 0; i < ND; ++i) c2f[i] = dir[i] != 0.0 ? 0.0 : invS[i] * (2.0 * m[k]);
#pragma unroll
        for (int i = 0; i < ND; ++i) {
            const double stp = (1.0 - neu[i]) * n[i] * (1.0 - c2f[i]);
            if (o.t[0]) o.t[0][at(ND, 1, i, r, 0)] = -(trm[i] * s);
            if (o.t[2]) o.t[2][at(ND, 1, i, r, 0)] = stp;
            if (o.t[5]) o.t[5][at(1, ND, 0, r, i)] = n[i] * c2f[i];
            if (o.t[7]) o.t[7][at(ND, 1, i, r, 0)] = pass[i] * c2f[i];
            if (o.t[9])
                o.t[9][at(ND, 1, i, r, 0)] = sA * invS[i] * (rob[i] * stp + neu[i] * (n[i] * c2f[i]));
        }
        if (o.t[6]) o.t[6][at(1, 1, 0, r, 0)] = -(dir_np * (A / ar_avg) * s);
        if constexpr (ND == 3) {
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
                for (int j = 0; j < 3; ++j) {
                    const double sr = -((1.0 - neu[i]) * R[i][j] * (1.0 - c2f[j]));
                    if (o.t[1]) o.t[1][at(3, 3, i, r, j)] = sr;
                    if (o.t[3]) o.t[3][at(3, 3, i, r, j)] = -(R[i][j] * c2f[j]);
                    if (o.t[4]) o.t[4][at(3, 3, i, r, j)] = -(pass[i] * d_rr * RR[i][j] * s);
                    if (o.t[8])
                        o.t[8][at(3, 3, i, r, j)] = sA * invS[i] * (rob[i] * sr - neu[i] * (R[i][j] * c2f[j]));
                }
        } else {
            double rr = 0.0;
#pragma unroll
            for (int i = 0; i < ND; ++i) {
                const double sr = -((1.0 - neu[i]) * v[i] * (1.0 - c2f[i]));
                if (o.t[1]) o.t[1][at(ND, 1, i, r, 0)] = sr;
                if (o.t[3]) o.t[3][at(1, ND, 0, r, i)] = v[i] * c2f[i];
                if (o.t[8]) o.t[8][at(ND, 1, i, r, 0)] = sA * invS[i] * (rob[i] * sr - neu[i] * (v[i] * c2f[i]));
                rr += (-v[i] * pass[i] * d_rr) * v[i];
            }
            if (o.t[4]) o.t[4][at(1, 1, 0, r, 0)] = -(rr * s);
        }
    }

    // face terms
#pragma unroll
    for (int j = 0; j < ND; ++j) {
        const double nm = invA * pass[j] * invS[j];
        const double q = (-nm - dir[j]) - b2f[j];
        if (o.t[10]) o.t[10][f * ND + j] = trm_bnd[j] * ssum;
        if (o.t[12]) o.t[12][f * ND + j] = n[j] * ((nm + dir[j]) + b2f[j]);
        if (o.t[13]) o.t[13][f * ND + j] = dir[j] + sA * invS[j] * (neu[j] + rob[j] * b2f[j]);
        if constexpr (ND == 3) {
#pragma unroll
            for (int i = 0; i < 3; ++i)
                if (o.t[11]) o.t[11][f * 9 + i * 3 + j] = R[i][j] * q;
        } else if (o.t[11]) {
            o.t[11][f * ND + j] = -v[j] * q;
        }
    }
}

}  // namespace pb
