// tpsa_system.cuh -- the linear system of the TPSA three-field elasticity model (reference models/momentum_balance.py:
// 82-106, 250-280, 344-368 with the fluxes of models/constitutive_laws.py:3064-3296), gathered per cell from the face
// values of tpsa_face.cuh:
//   momentum     -div_nd (S_u u + S_r r + S_p p + B_s g)               - f   = 0
//   angular      -vol/mu r + div_nr (R_u u + R_r r + B_r g)            - s_r = 0
//   solid mass   -vol/lambda p + div (M_u u + M_p p + B_m g)           - s_p = 0
// Unknowns and equations are numbered cell by cell, [u_c (nd), r_c (nr), p_c (1)], so the diagonal blocks of A are the
// cell blocks.  Block (c, k) exists for k = c and every face neighbour k of c; of its (nd+nr+1)^2 entries only the
// structurally non-zero ones are stored (u-u is diagonal, r-p and p-r are zero): 37 of 49 in 3-D, 12 of 16 in 2-D.
// Each block (c, k) is written by one thread (or one host loop step) that walks the faces of c, so there are no atomics
// and two assemblies are bit-identical.  The CUDA kernels are in face.cu; the test-only host build in tests/emu.
#pragma once
#include <cstdint>

#include "views.hpp"

namespace pb {

// neighbours per cell (the cell itself included) the pattern supports
constexpr int kTpsaMaxNb = 32;

// Layout of one block row.  Row l of a cell: l < ND displacement component l, then NR rotation rows, then the total
// pressure row.  Per neighbour a row holds len(l) entries, neighbours in ascending cell order; inside one neighbour k
// the columns are ascending: u row i -> [u_i, r_0 .. r_NR-1, p], r row -> [u_0 .. u_ND-1, r_0 .. r_NR-1],
// p row -> [u_0 .. u_ND-1, p].  Block row c starts at NZ * cc_ptr[c]; row l at NZ * cc_ptr[c] + off(l) * n_c.
template <int ND>
struct TpsaDims {
    static constexpr int NR = ND == 3 ? 3 : 1, B = ND + NR + 1;
    static constexpr int LU = NR + 2, LR = ND + NR, LP = ND + 1;
    static constexpr int NZ = ND * LU + NR * LR + LP;
    PB_HD static int len(int l) { return l < ND ? LU : (l < ND + NR ? LR : LP); }
    PB_HD static int off(int l) { return l < ND ? l * LU : (l < ND + NR ? ND * LU + (l - ND) * LR : ND * LU + NR * LR); }
    // column, relative to k * B, of entry t of row l
    PB_HD static int col(int l, int t) {
        if (l < ND) return t == 0 ? l : (t <= NR ? ND + t - 1 : ND + NR);
        if (l < ND + NR) return t;
        return t < ND ? t : ND + NR;
    }
};

// cell -> face lists (cell_faces in CSC form) and the face -> cell table of face.cu: 2 per face, (cell << 1) | (sign <
// 0), -1 = none; fc_ptr[f] = first (face, cell) entry of face f in the value layouts of tpsa_face.cuh
struct TpsaTopo {
    int64_t nc;
    const int32_t *cf_ip, *cf_ix;
    const int32_t *face_cells;
    const int32_t *fc_ptr;
};

// The distinct cells sharing a face with c, c included, ascending, into nb; returns their number, or -1 when there
// are more than kTpsaMaxNb.
PB_HD int tpsa_cell_neighbours(int64_t c, const TpsaTopo &t, int32_t *nb) {
    int n = 1;
    nb[0] = (int32_t)c;
    for (int q = t.cf_ip[c]; q < t.cf_ip[c + 1]; ++q) {
        const int64_t f = t.cf_ix[q];
        for (int sd = 0; sd < 2; ++sd) {
            const int32_t e = t.face_cells[2 * f + sd];
            if (e < 0) continue;
            const int32_t k = e >> 1;
            int pos = 0;
            while (pos < n && nb[pos] < k) ++pos;
            if (pos < n && nb[pos] == k) continue;
            if (n == kTpsaMaxNb) return -1;
            for (int i = n; i > pos; --i) nb[i] = nb[i - 1];
            nb[pos] = k;
            ++n;
        }
    }
    return n;
}

// Row pointers and column indices of block row c (n = its neighbour count, nb = its neighbours).
template <int ND>
PB_HD void tpsa_pattern_rows(int64_t c, int n, const int32_t *nb, int64_t cc0, int32_t *ip, int32_t *ix) {
    using D = TpsaDims<ND>;
    const int64_t base = (int64_t)D::NZ * cc0;
    for (int l = 0; l < D::B; ++l) {
        const int len = D::len(l);
        const int64_t r0 = base + (int64_t)D::off(l) * n;
        ip[c * D::B + l] = (int32_t)r0;
        for (int j = 0; j < n; ++j)
            for (int t = 0; t < len; ++t) ix[r0 + j * len + t] = nb[j] * D::B + D::col(l, t);
    }
}

// face values the system reads (PB_TPSA_* order of include/poreb200.h: 0-6 cell terms, 10-12 boundary terms)
struct TpsaTerms {
    const double *t[14];
};

// Entries of row l of block row c in block (c, k), k a neighbour of c (or c itself): the len(l) values at dst.  Every entry sums the faces of c in the order of its cell -> face list, so the values do not depend on how the
// work is split.
template <int ND>
PB_HD void tpsa_system_segment(int64_t c, int l, int64_t k, const TpsaTopo &t, const TpsaTerms &T, const double *mu,
                               const double *lam, const double *vol, double *dst) {
    using D = TpsaDims<ND>;
    constexpr int NR = D::NR, LMAX = D::LR > D::LU ? D::LR : D::LU;
    double acc[LMAX];
#pragma unroll
    for (int q = 0; q < LMAX; ++q) acc[q] = 0.0;
    for (int q = t.cf_ip[c]; q < t.cf_ip[c + 1]; ++q) {
        const int64_t f = t.cf_ix[q];
        const int32_t e0 = t.face_cells[2 * f], e1 = t.face_cells[2 * f + 1];
        const int L = e1 >= 0 ? 2 : 1;
        const int64_t c0 = e0 >> 1, c1 = e1 >= 0 ? (int64_t)(e1 >> 1) : -1;
        if (c0 != k && c1 != k) continue;
        const double s = (((c0 == c) ? e0 : e1) & 1) ? -1.0 : 1.0;   // cell_faces[f, c]: div = cell_faces^T
        const int r = (L == 2 && (c0 == k ? c1 : c0) < k) ? 1 : 0;    // rank of k among the face's cells
        const int64_t p0 = t.fc_ptr[f];
        if (l < ND) {
            const int i = l;
            acc[0] -= s * T.t[0][ND * p0 + i * L + r];
#pragma unroll
            for (int m = 0; m < NR; ++m) acc[1 + m] -= s * T.t[1][ND * NR * p0 + i * NR * L + r * NR + m];
            acc[1 + NR] -= s * T.t[2][ND * p0 + i * L + r];
        } else if (l < ND + NR) {
            const int i = l - ND;
#pragma unroll
            for (int m = 0; m < ND; ++m) acc[m] += s * T.t[3][NR * ND * p0 + i * ND * L + r * ND + m];
#pragma unroll
            for (int m = 0; m < NR; ++m) acc[ND + m] += s * T.t[4][NR * NR * p0 + i * NR * L + r * NR + m];
        } else {
#pragma unroll
            for (int m = 0; m < ND; ++m) acc[m] += s * T.t[5][ND * p0 + r * ND + m];
            acc[ND] += s * T.t[6][p0 + r];
        }
    }
    if (k == c && l >= ND) {
        if (l < ND + NR) acc[l] -= vol[c] / mu[c];    // r row i: column r_i is entry ND + i == l
        else acc[ND] -= vol[c] / lam[c];
    }
    const int len = D::len(l);
#pragma unroll
    for (int q = 0; q < LMAX; ++q)
        if (q < len) dst[q] = acc[q];
}

// Block (c, cc_ix[j0 + j]) of A, all rows, into the CSR values a (j0 = cc_ptr[c], n neighbours).
template <int ND>
PB_HD void tpsa_system_block(int64_t c, int j, const TpsaTopo &t, const int32_t *cc_ptr, const int32_t *cc_ix,
                             const TpsaTerms &T, const double *mu, const double *lam, const double *vol, double *a) {
    using D = TpsaDims<ND>;
    const int64_t j0 = cc_ptr[c];
    const int n = (int)(cc_ptr[c + 1] - j0);
    const int64_t k = cc_ix[j0 + j];
#pragma unroll
    for (int l = 0; l < D::B; ++l)
        tpsa_system_segment<ND>(c, l, k, t, T, mu, lam, vol,
                                a + (int64_t)D::NZ * j0 + (int64_t)D::off(l) * n + (int64_t)j * D::len(l));
}

// Entry l of block c of b = -R(0):  div_nd B_s g + f,  -div_nr B_r g + s_r,  -div B_m g + s_p.  g: nd values per face
// at f*nd + i; src: the f / s_r / s_p entry of this row (0 when not given).
template <int ND>
PB_HD double tpsa_rhs_row(int64_t c, int l, const TpsaTopo &t, const TpsaTerms &T, const double *g, double src) {
    constexpr int NR = TpsaDims<ND>::NR;
    double acc = 0.0;
    for (int q = t.cf_ip[c]; q < t.cf_ip[c + 1]; ++q) {
        const int64_t f = t.cf_ix[q];
        const int32_t e0 = t.face_cells[2 * f], e1 = t.face_cells[2 * f + 1];
        const double s = ((((int64_t)(e0 >> 1) == c) ? e0 : e1) & 1) ? -1.0 : 1.0;
        const double *gf = g + f * ND;
        if (l < ND) {
            acc += s * (T.t[10][f * ND + l] * gf[l]);
        } else {
            const double *w = l < ND + NR ? T.t[11] + f * NR * ND + (l - ND) * ND : T.t[12] + f * ND;
            double v = 0.0;
#pragma unroll
            for (int m = 0; m < ND; ++m) v += w[m] * gf[m];
            acc -= s * v;
        }
    }
    return acc + src;
}

// ---- TPSA poromechanics and thermo-poromechanics (reference models/poromechanics.py:92-136, 177-213) --------------
// Unknowns and equations per cell [u_c (nd), r_c (nr), p_t_c, s_c (NS)]: NS scalar balances after the total pressure,
// s = [p] for poromechanics (NS = 1) and [p, T] for thermo-poromechanics (NS = 2), so B = nd + nr + 1 + NS (5 / 8 and
// 6 / 9).  The mechanics rows are the three-field rows (columns relative to k * B) with the solid-mass row extended by
// the fluid pressure: [u_0 .. u_ND-1, p_t, p] per neighbour k, whose p entry is -vol alpha / lambda for k = c and 0
// otherwise; they have no T column (the TPSA stress of the reference has no thermal term).  Scalar row s of c holds the
// whole own block [u_c, r_c, p_t_c, s_c] and the NS scalar columns of every other cell in row c of the flux pattern
// (div @ flux, MPFA; with NS = 2 the union of the Darcy and Fourier patterns), ascending.  Block row c starts at
// blk_ptr[c]: the mechanics rows first, row l at blk_ptr[c] + off(l) * n_c, then scalar row s at
// blk_ptr[c] + NZ * n_c + s * (B + NS * m_c), m_c the other cells of the flux-pattern row.
template <int ND, int NS = 1>
struct TpsaPoroDims {
    using M = TpsaDims<ND>;
    static constexpr int NR = M::NR, B = M::B + NS, LP = M::LP + 1;
    static constexpr int NZ = ND * M::LU + NR * M::LR + LP;   // mechanics entries per neighbour
    PB_HD static int len(int l) { return l < ND + NR ? M::len(l) : LP; }
    PB_HD static int off(int l) { return M::off(l); }
    PB_HD static int col(int l, int t) { return l < ND + NR ? M::col(l, t) : (t < ND ? t : ND + NR + (t - ND)); }
};

// Entries of block row c in the fixed pattern: NZ per face neighbour, and per scalar row B for the own block and NS per
// other cell of row c of the flux pattern (fp_*: sorted CSR).
template <int ND, int NS = 1>
PB_HD int64_t tpsa_poro_row_count(int64_t c, int n, const int32_t *fp_ip, const int32_t *fp_ix) {
    using D = TpsaPoroDims<ND, NS>;
    int64_t m = 0;
    for (int q = fp_ip[c]; q < fp_ip[c + 1]; ++q) m += fp_ix[q] != c;
    return (int64_t)D::NZ * n + NS * (D::B + NS * m);
}

// Row pointers and column indices of block row c (n face neighbours nb, ascending; the block row starts at blk0).
template <int ND, int NS = 1>
PB_HD void tpsa_poro_pattern_rows(int64_t c, int n, const int32_t *nb, int64_t blk0, const int32_t *fp_ip,
                                  const int32_t *fp_ix, int32_t *ip, int32_t *ix) {
    using D = TpsaPoroDims<ND, NS>;
    constexpr int MB = D::M::B;   // mechanics rows per cell; scalar s sits at column MB + s of a block
    for (int l = 0; l < MB; ++l) {
        const int len = D::len(l);
        const int64_t r0 = blk0 + (int64_t)D::off(l) * n;
        ip[c * D::B + l] = (int32_t)r0;
        for (int j = 0; j < n; ++j)
            for (int t = 0; t < len; ++t) ix[r0 + j * len + t] = nb[j] * D::B + D::col(l, t);
    }
    int64_t q0 = blk0 + (int64_t)D::NZ * n;
    for (int s = 0; s < NS; ++s) {
        ip[c * D::B + MB + s] = (int32_t)q0;
        bool own = false;
        for (int q = fp_ip[c]; q <= fp_ip[c + 1]; ++q) {
            const int32_t k = q < fp_ip[c + 1] ? fp_ix[q] : INT32_MAX;
            if (!own && k >= c) {
                for (int t = 0; t < D::B; ++t) ix[q0++] = (int32_t)(c * D::B + t);
                own = true;
            }
            if (k != c && k != INT32_MAX)
                for (int u = 0; u < NS; ++u) ix[q0++] = k * D::B + MB + u;
        }
    }
}

// Mechanics rows of block (c, cc_ix[j0 + j]) into the CSR values a; thread j = 0 also zeroes the scalar rows of c.
template <int ND, int NS = 1>
PB_HD void tpsa_poro_block(int64_t c, int j, const TpsaTopo &t, const int32_t *cc_ptr, const int32_t *cc_ix,
                           const int64_t *blk_ptr, const TpsaTerms &T, const double *mu, const double *lam,
                           const double *alpha, const double *vol, double *a) {
    using D = TpsaPoroDims<ND, NS>;
    constexpr int MB = D::M::B;
    const int64_t j0 = cc_ptr[c];
    const int n = (int)(cc_ptr[c + 1] - j0);
    const int64_t k = cc_ix[j0 + j];
    const int64_t b0 = blk_ptr[c];
#pragma unroll
    for (int l = 0; l < MB; ++l) {
        double *dst = a + b0 + (int64_t)D::off(l) * n + (int64_t)j * D::len(l);
        tpsa_system_segment<ND>(c, l, k, t, T, mu, lam, vol, dst);
        if (l == MB - 1) dst[ND + 1] = k == c ? -vol[c] * alpha[c] / lam[c] : 0.0;
    }
    if (j == 0)
        for (int64_t q = b0 + (int64_t)D::NZ * n; q < blk_ptr[c + 1]; ++q) a[q] = 0.0;
}

// Scalar rows of cell c at one Newton step: row s * nc + c of the field-ordered Jacobian jf (NS nc rows, columns
// [p_t (nc) | s_0 (nc) .. s_NS-1 (nc)]) placed into the fixed pattern of scalar row s (sorted, from row0 = the first
// scalar row of c; binary search per entry, duplicates summed in row order), and -R into b[c * B + MB + s].  Returns
// the number of entries that are not in the pattern (0 by construction).
template <int ND, int NS = 1>
PB_HD int tpsa_poro_fluid_row(int64_t c, int64_t nc, const int64_t *blk_ptr, int64_t row0, const int32_t *ix,
                              const int32_t *jf_ip, const int32_t *jf_ix, const double *jf_a, const double *neg_res,
                              double *a, double *b) {
    using D = TpsaPoroDims<ND, NS>;
    constexpr int MB = D::M::B;
    const int64_t len = (blk_ptr[c + 1] - row0) / NS;
    int missing = 0;
    for (int s = 0; s < NS; ++s) {
        const int64_t s0 = row0 + s * len, e = s0 + len, r = s * nc + c;
        for (int64_t q = s0; q < e; ++q) a[q] = 0.0;
        for (int q = jf_ip[r]; q < jf_ip[r + 1]; ++q) {
            int64_t col = jf_ix[q];
            int fld = 0;   // 0: p_t, 1 + u: scalar u
            while (fld < NS && col >= nc) { col -= nc; ++fld; }
            const int32_t want = (int32_t)(col * D::B + MB - 1 + fld);
            int64_t lo = s0, hi = e;
            while (lo < hi) {
                const int64_t mid = (lo + hi) >> 1;
                if (ix[mid] < want) lo = mid + 1; else hi = mid;
            }
            if (lo < e && ix[lo] == want) a[lo] += jf_a[q];
            else ++missing;
        }
        b[c * D::B + MB + s] = neg_res[r];
    }
    return missing;
}

// ---- TPSA elasticity with fractures in frictional contact (reference models/momentum_balance.py:127-183,
// constitutive_laws.py:3064-3248, contact_mechanics.py:80-245) -----------------------------------------------------
// Unknowns [three-field cell blocks (B nc) | t (nd per fracture cell, nk) | u_j (nd per mortar cell, nm)]; equations
// [three-field balances (B nc) | interface force balances (nd per mortar cell) | normal laws (nk) | tangential laws
// ((nd - 1) nk)].  Fracture cells and mortar cells are numbered over all fractures / interfaces one after the other.
// The fracture faces of the matrix are internal Dirichlet faces carrying Pi^avg u_j, so the balance rows of a cell with
// fracture faces gain u_j columns after the three-field segments: block row c holds, per row l, the n len(l) entries of
// its face neighbours, then per fracture face (mortar cells ascending) one u_j entry in a momentum row and nd in an
// angular or solid-mass row:
//   momentum i   -s_f B_s[f, i] w_m2p      angular  +s_f B_r[f, :, :] w_m2p      solid mass  +s_f B_m[f, :] w_m2p
// Block row c starts at blk_ptr[c], row l at blk_ptr[c] + off(l) n_c + eoff(l) m_c (m_c: fracture faces of c).  The
// force row (M, i) (face f, cell c, fracture cell K) has LF entries, at blk_ptr[nc] + (M nd + i) LF:
//   [u_c,i | r_c | p_c]  w_p2m s_f (S_u | S_r | S_p)[f, i],   t_K  vol_M T_c sign_M R_K[:, i],   u_j(M, i)  w_p2m s_f B_s w_m2p
// and contact row r (r < nk: the normal law of K = r, else a tangential law of K = (r - nk) / (nd - 1)) the 3 nd
// columns [t_K | u_j(m1) | u_j(m2)] (m1 < m2 the mortar cells of K), at blk_ptr[nc] + nm nd LF + 3 nd r.
struct TpsaMortars {
    int64_t nm, nk;
    const int32_t *face, *cell, *face_mortar, *pair;   // pair: the two mortar cells of every fracture cell, ascending
    const double *w_m2p, *w_p2m, *sign, *vol, *frame;   // vol: volume x secondary_to_mortar_int weight; frame: nd x nd
    double ct;                                           // per fracture cell, row-major (tangents, then the normal)
};

template <int ND>
struct TpsaContactDims {
    using M = TpsaDims<ND>;
    static constexpr int NR = M::NR, B = M::B, LF = ND + NR + 3, LC = 3 * ND;
    static constexpr int EXT = ND + NR * ND + ND;   // u_j entries of one fracture face in a block row
    PB_HD static int ext(int l) { return l < ND ? 1 : ND; }
    PB_HD static int eoff(int l) { return l < ND ? l : ND + (l - ND) * ND; }
    PB_HD static int64_t roff(int l, int n, int m) { return (int64_t)M::off(l) * n + (int64_t)eoff(l) * m; }
};

// Fracture faces of c (faces with a mortar cell).
PB_HD int tpsa_contact_nfrac(int64_t c, const TpsaTopo &t, const int32_t *face_mortar) {
    int m = 0;
    for (int q = t.cf_ip[c]; q < t.cf_ip[c + 1]; ++q) m += face_mortar[t.cf_ix[q]] >= 0;
    return m;
}

// The fracture face of c with the smallest mortar cell above `last` (-1: from the start); its mortar cell, or -1.
PB_HD int32_t tpsa_contact_next(int64_t c, const TpsaTopo &t, const int32_t *face_mortar, int32_t last, int64_t *face) {
    int32_t best = -1;
    for (int q = t.cf_ip[c]; q < t.cf_ip[c + 1]; ++q) {
        const int64_t f = t.cf_ix[q];
        const int32_t m = face_mortar[f];
        if (m > last && (best < 0 || m < best)) { best = m; *face = f; }
    }
    return best;
}

// Row pointers and column indices of block row c (n face neighbours nb, ascending; the block row starts at blk0).
template <int ND>
PB_HD void tpsa_contact_pattern_rows(int64_t c, int n, const int32_t *nb, int64_t blk0, const TpsaTopo &t,
                                     const TpsaMortars &I, int32_t *ip, int32_t *ix) {
    using D = TpsaContactDims<ND>;
    const int m = tpsa_contact_nfrac(c, t, I.face_mortar);
    const int64_t u0 = (int64_t)D::B * t.nc + (int64_t)ND * I.nk;
    for (int l = 0; l < D::B; ++l) {
        const int len = D::M::len(l);
        const int64_t r0 = blk0 + D::roff(l, n, m);
        ip[c * D::B + l] = (int32_t)r0;
        for (int j = 0; j < n; ++j)
            for (int q = 0; q < len; ++q) ix[r0 + j * len + q] = nb[j] * D::B + D::M::col(l, q);
        int64_t q = r0 + (int64_t)n * len, f = 0;
        for (int32_t mc = tpsa_contact_next(c, t, I.face_mortar, -1, &f); mc >= 0;
             mc = tpsa_contact_next(c, t, I.face_mortar, mc, &f)) {
            if (l < ND) ix[q++] = (int32_t)(u0 + (int64_t)mc * ND + l);
            else
                for (int i = 0; i < ND; ++i) ix[q++] = (int32_t)(u0 + (int64_t)mc * ND + i);
        }
    }
}

// Row pointer and column indices of interface row q (q < nd nm: force row (q / nd, q % nd); else contact row
// q - nd nm); the interface rows start at row0 = B nc and entry e0 = blk_ptr[nc].
template <int ND>
PB_HD void tpsa_contact_iface_pattern(int64_t q, int64_t nc, int64_t e0, const TpsaTopo &t, const TpsaMortars &I,
                                      int32_t *ip, int32_t *ix) {
    using D = TpsaContactDims<ND>;
    const int64_t t0 = (int64_t)D::B * nc, u0 = t0 + (int64_t)ND * I.nk;
    if (q < ND * I.nm) {
        const int64_t mc = q / ND, f = I.face[mc];
        const int i = (int)(q - mc * ND);
        const int64_t c = t.face_cells[2 * f] >> 1, k = I.cell[mc];
        int64_t p = e0 + q * D::LF;
        ip[t0 + q] = (int32_t)p;
        ix[p++] = (int32_t)(c * D::B + i);
        for (int r = 0; r <= D::NR; ++r) ix[p++] = (int32_t)(c * D::B + ND + r);
        for (int j = 0; j < ND; ++j) ix[p++] = (int32_t)(t0 + k * ND + j);
        ix[p] = (int32_t)(u0 + mc * ND + i);
    } else {
        const int64_t r = q - ND * I.nm;
        const int64_t k = r < I.nk ? r : (r - I.nk) / (ND - 1);
        int64_t p = e0 + (int64_t)ND * I.nm * D::LF + r * D::LC;
        ip[t0 + q] = (int32_t)p;
        for (int j = 0; j < ND; ++j) ix[p++] = (int32_t)(t0 + k * ND + j);
        for (int s = 0; s < 2; ++s)
            for (int j = 0; j < ND; ++j) ix[p++] = (int32_t)(u0 + (int64_t)I.pair[2 * k + s] * ND + j);
    }
}

// Block (c, cc_ix[j0 + j]) of the balance rows into the CSR values a; thread j = 0 also writes the u_j entries of c.
template <int ND>
PB_HD void tpsa_contact_block(int64_t c, int j, const TpsaTopo &t, const int32_t *cc_ptr, const int32_t *cc_ix,
                              const int64_t *blk_ptr, const TpsaMortars &I, const TpsaTerms &T, const double *mu,
                              const double *lam, const double *vol, double *a) {
    using D = TpsaContactDims<ND>;
    constexpr int NR = D::NR;
    const int64_t j0 = cc_ptr[c];
    const int n = (int)(cc_ptr[c + 1] - j0);
    const int64_t k = cc_ix[j0 + j];
    const int m = tpsa_contact_nfrac(c, t, I.face_mortar);
    const int64_t b0 = blk_ptr[c];
#pragma unroll
    for (int l = 0; l < D::B; ++l)
        tpsa_system_segment<ND>(c, l, k, t, T, mu, lam, vol, a + b0 + D::roff(l, n, m) + (int64_t)j * D::M::len(l));
    if (j != 0 || m == 0) return;
    int64_t f = 0;
    int e = 0;   // fracture faces of c done
    for (int32_t mc = tpsa_contact_next(c, t, I.face_mortar, -1, &f); mc >= 0;
         mc = tpsa_contact_next(c, t, I.face_mortar, mc, &f), ++e) {
        const double s = (t.face_cells[2 * f] & 1) ? -1.0 : 1.0, w = s * I.w_m2p[mc];
#pragma unroll
        for (int l = 0; l < D::B; ++l) {
            double *dst = a + b0 + D::roff(l, n, m) + (int64_t)n * D::M::len(l) + (int64_t)e * D::ext(l);
            if (l < ND) {
                dst[0] = -w * T.t[10][f * ND + l];
            } else if (l < ND + NR) {
#pragma unroll
                for (int i = 0; i < ND; ++i) dst[i] = w * T.t[11][f * NR * ND + (l - ND) * ND + i];
            } else {
#pragma unroll
                for (int i = 0; i < ND; ++i) dst[i] = w * T.t[12][f * ND + i];
            }
        }
    }
}

// Values of interface row q (see tpsa_contact_iface_pattern): the force rows, 0 in the contact rows.
template <int ND>
PB_HD void tpsa_contact_iface_row(int64_t q, int64_t e0, const TpsaTopo &t, const TpsaMortars &I, const TpsaTerms &T,
                                  double *a) {
    using D = TpsaContactDims<ND>;
    constexpr int NR = D::NR;
    if (q < ND * I.nm) {
        const int64_t mc = q / ND, f = I.face[mc], k = I.cell[mc];
        const int i = (int)(q - mc * ND);
        const double w = ((t.face_cells[2 * f] & 1) ? -1.0 : 1.0) * I.w_p2m[mc];
        const int64_t p0 = t.fc_ptr[f];   // the face's one (face, cell) entry
        double *dst = a + e0 + q * D::LF;
        dst[0] = w * T.t[0][ND * p0 + i];
#pragma unroll
        for (int r = 0; r < NR; ++r) dst[1 + r] = w * T.t[1][ND * NR * p0 + i * NR + r];
        dst[1 + NR] = w * T.t[2][ND * p0 + i];
        const double tw = I.vol[mc] * I.ct * I.sign[mc];
#pragma unroll
        for (int j = 0; j < ND; ++j) dst[2 + NR + j] = tw * I.frame[k * ND * ND + j * ND + i];
        dst[2 + NR + ND] = w * T.t[10][f * ND + i] * I.w_m2p[mc];
    } else {
        double *dst = a + e0 + (int64_t)ND * I.nm * D::LF + (q - ND * I.nm) * D::LC;
#pragma unroll
        for (int p = 0; p < D::LC; ++p) dst[p] = 0.0;
    }
}

// Entry q of b = -R(0) for q >= B nc (interface rows): -w_p2m s_f B_s[f, i] g[f, i] in the force rows, 0 in the
// contact rows (written at every linearization).
template <int ND>
PB_HD double tpsa_contact_iface_rhs(int64_t q, const TpsaTopo &t, const TpsaMortars &I, const TpsaTerms &T,
                                    const double *g) {
    if (q >= ND * I.nm) return 0.0;
    const int64_t mc = q / ND, f = I.face[mc];
    const int i = (int)(q - mc * ND);
    const double s = (t.face_cells[2 * f] & 1) ? -1.0 : 1.0;
    return -I.w_p2m[mc] * s * T.t[10][f * ND + i] * g[f * ND + i];
}

// Contact row r at one Newton step: row r of jc (the Jacobian of the laws in the variables [t | u_j]) placed into the
// fixed pattern at its column + B nc (binary search, duplicates summed in row order), -R into b[row].  Returns the
// number of entries that are not in the pattern.
template <int ND>
PB_HD int tpsa_contact_law_row(int64_t r, int64_t c0, int64_t e0, int64_t row, const int32_t *ix, const int32_t *jc_ip,
                               const int32_t *jc_ix, const double *jc_a, const double *neg_res, double *a, double *b) {
    constexpr int LC = TpsaContactDims<ND>::LC;
    const int64_t s0 = e0 + r * LC, e = s0 + LC;   // e0: the first entry of the contact rows
    int missing = 0;
    for (int64_t q = s0; q < e; ++q) a[q] = 0.0;
    for (int q = jc_ip[r]; q < jc_ip[r + 1]; ++q) {
        const int32_t want = (int32_t)(jc_ix[q] + c0);
        int64_t lo = s0, hi = e;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (ix[mid] < want) lo = mid + 1; else hi = mid;
        }
        if (lo < e && ix[lo] == want) a[lo] += jc_a[q];
        else ++missing;
    }
    b[row] = neg_res[r];
    return missing;
}

}  // namespace pb
