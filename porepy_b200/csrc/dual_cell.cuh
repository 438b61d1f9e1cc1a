// dual_cell.cuh -- per-(cell, local face) routines of the two mixed (dual) discretizations of Darcy flow: the lowest
// order mixed virtual element method (reference numerics/vem/mvem.py, MVEM.massHdiv and cell_diameters of
// grids/grid.py) and the lowest order Raviart-Thomas element (numerics/fem/rt0.py, RT0.massHdiv, faces_to_cell and
// _compute_cell_face_to_opposite_node).  One call computes row i of the local mass matrix of cell c and hands it to a
// row sink: DualScatter adds it into the global FACE x FACE values and writes column i of the cell's (3 x n_faces)
// flux reconstruction, with nothing staged per cell, so polyhedra with any number of faces need no local arrays;
// DualLocalRow writes it into row i of a per-cell buffer for the hybridization (dual_hybrid.cuh).  The CUDA kernel
// dual_kernel (dual.cu) runs one thread per entry of cell_faces with DualScatter; the test-only host build loops.
#pragma once
#include <cmath>
#include <cstdint>

#include "views.hpp"

namespace pb {

enum { kDualMvem = 0, kDualRt0 = 1 };

// Topology: cell_faces as CSC (cf_ip / cf_ix / cf_sg, the faces of every cell sorted), cf_cell[q] = cell of entry q,
// face_nodes as CSC, and the FACE x FACE mass pattern (row f: every face sharing a cell with f, sorted).
struct DualTopo {
    const int32_t *cf_ip, *cf_ix, *cf_cell;
    const int8_t *cf_sg;
    const int32_t *fn_ip, *fn_ix, *mass_ip, *mass_ix;
};

// Geometry in the grid's own frame, each array (3, n) row-major: component k of entity e at k * n + e.  Only the first
// ND components enter the schemes; the cell diameter uses all three (any rotation keeps distances).
// perm: (3, 3, nc) row-major, the tensor already expressed in the frame.  rot: the frame's 3 x 3 rotation (rows =
// the frame's axes), used to bring the flux reconstruction back to the ambient space.
struct DualGeo {
    int64_t nn, nf, nc;
    const double *nodes, *fnorm, *fcent, *ccent, *vol, *perm, *rot;
};

// Two cells at most add to one mass entry, each once, into a zeroed value: the sum is the same double in either
// order, so repeats are bit-identical.
PB_HD void dual_add(double *p, double v) {
#ifdef __CUDA_ARCH__
    atomicAdd(p, v);
#else
    *p += v;
#endif
}

template <int ND>
PB_HD void dual_perm(const DualGeo &G, int64_t c, double K[ND][ND]) {
    for (int a = 0; a < ND; ++a)
        for (int b = 0; b < ND; ++b) K[a][b] = G.perm[(a * 3 + b) * G.nc + c];
}

// Inverse of the symmetric tensor by the reference's explicit formulas (dual_elliptic.py _inv_matrix_{1,2,3}d).
template <int ND>
PB_HD void dual_inv(const double K[ND][ND], double Ki[ND][ND]) {
    if constexpr (ND == 1) {
        Ki[0][0] = 1.0 / K[0][0];
    } else if constexpr (ND == 2) {
        const double det = K[0][0] * K[1][1] - K[0][1] * K[0][1];
        Ki[0][0] = K[1][1] / det; Ki[0][1] = -K[0][1] / det;
        Ki[1][0] = -K[0][1] / det; Ki[1][1] = K[0][0] / det;
    } else {
        const double det = K[0][0] * K[1][1] * K[2][2] - K[0][0] * K[1][2] * K[1][2] - K[0][1] * K[0][1] * K[2][2] +
                           2 * K[0][1] * K[0][2] * K[1][2] - K[0][2] * K[0][2] * K[1][1];
        Ki[0][0] = (K[1][1] * K[2][2] - K[1][2] * K[1][2]) / det;
        Ki[0][1] = (K[0][2] * K[1][2] - K[0][1] * K[2][2]) / det;
        Ki[0][2] = (K[0][1] * K[1][2] - K[0][2] * K[1][1]) / det;
        Ki[1][0] = (K[0][2] * K[1][2] - K[0][1] * K[2][2]) / det;
        Ki[1][1] = (K[0][0] * K[2][2] - K[0][2] * K[0][2]) / det;
        Ki[1][2] = (K[0][2] * K[1][0] - K[0][0] * K[1][2]) / det;
        Ki[2][0] = (K[0][1] * K[1][2] - K[0][2] * K[1][1]) / det;
        Ki[2][1] = (K[0][1] * K[0][2] - K[0][0] * K[1][2]) / det;
        Ki[2][2] = (K[0][0] * K[1][1] - K[0][1] * K[0][1]) / det;
    }
}

// Largest distance between two nodes of cell c (grid.py cell_diameters), over the nodes of its faces.
PB_HD double dual_diameter(const DualTopo &T, const DualGeo &G, int64_t c) {
    double d2 = 0.0;
    for (int q = T.cf_ip[c]; q < T.cf_ip[c + 1]; ++q) {
        const int32_t f = T.cf_ix[q];
        for (int r = T.fn_ip[f]; r < T.fn_ip[f + 1]; ++r) {
            const int32_t a = T.fn_ix[r];
            for (int q2 = q; q2 < T.cf_ip[c + 1]; ++q2) {
                const int32_t f2 = T.cf_ix[q2];
                for (int r2 = T.fn_ip[f2]; r2 < T.fn_ip[f2 + 1]; ++r2) {
                    const int32_t b = T.fn_ix[r2];
                    double s = 0.0;
                    for (int k = 0; k < 3; ++k) {
                        const double t = G.nodes[k * G.nn + a] - G.nodes[k * G.nn + b];
                        s += t * t;
                    }
                    d2 = s > d2 ? s : d2;
                }
            }
        }
    }
    return sqrt(d2);
}

// Position of column j in mass row f (binary search; the column is in the pattern by construction).
PB_HD int32_t dual_pos(const DualTopo &T, int32_t f, int32_t j) {
    int32_t lo = T.mass_ip[f], hi = T.mass_ip[f + 1];
    while (lo < hi) {
        const int32_t mid = (lo + hi) >> 1;
        if (T.mass_ix[mid] < j) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// Row sink of dual_kernel: mass entry (row fi, column face of entry qj) added into the global values, flux
// reconstruction column written to proj.
struct DualScatter {
    double *mass, *proj;
    PB_HD void entry(const DualTopo &T, int32_t fi, int qj, double v) const {
        dual_add(mass + dual_pos(T, fi, T.cf_ix[qj]), v);
    }
    // MVEM entry: consistency part and weighted stabilization, F_i^T G^-1 F_j + w stab
    PB_HD void mvem_entry(const DualTopo &T, int32_t fi, int qj, double cons, double w, double stab) const {
        dual_add(mass + dual_pos(T, fi, T.cf_ix[qj]), cons + w * stab);
    }
    template <int ND>
    PB_HD void column(const DualTopo &T, const DualGeo &G, int64_t c, int i, const double p[ND]) const;
};

// Row sink of the hybridization: row i of the cell's local matrix in outward-flux variables, s_i s_j A_ij (hybrid.py
// passes outward normals and unit signs to massHdiv), at row[j] for the j-th face of the cell.  inv_a = 1 / aperture:
// hybrid.py scales the cell volume and the normals by the aperture, which divides the consistency part by it and
// leaves the stabilization unchanged.  No flux reconstruction.
struct DualLocalRow {
    double *row;
    double si, inv_a;
    int b;   // cf_ip[c]
    PB_HD void entry(const DualTopo &T, int32_t, int qj, double v) const { row[qj - b] = si * (double)T.cf_sg[qj] * v; }
    PB_HD void mvem_entry(const DualTopo &T, int32_t, int qj, double cons, double w, double stab) const {
        row[qj - b] = si * (double)T.cf_sg[qj] * (cons * inv_a + w * stab);
    }
    template <int ND>
    PB_HD void column(const DualTopo &, const DualGeo &, int64_t, int, const double *) const {}
};

// Flux reconstruction column: proj row 3c + a holds the faces of c in cell_faces order, at 3 cf_ip[c] + a n + i.
template <int ND>
PB_HD void dual_proj_column(const DualTopo &T, const DualGeo &G, int64_t c, int i, const double p[ND], double *proj) {
    const int b = T.cf_ip[c], n = T.cf_ip[c + 1] - b;
    for (int a = 0; a < 3; ++a) {
        double s = 0.0;
        for (int k = 0; k < ND; ++k) s += G.rot[k * 3 + a] * p[k];
        proj[3 * (int64_t)b + a * n + i] = s;
    }
}

template <int ND>
PB_HD void DualScatter::column(const DualTopo &T, const DualGeo &G, int64_t c, int i, const double p[ND]) const {
    dual_proj_column<ND>(T, G, c, i, p, proj);
}

// MVEM row, with diam the cell diameter, s_j the sign and x_j, n_j the centre and normal of face j:
//   D_j = K^T n_j / diam, F_j = s_j (x_j - x_c) / diam, G = K vol / diam^2, Pi_j = G^-1 F_j,
//   A_ij = F_i^T G^-1 F_j + w sum_k (delta_ki - D_k.Pi_i)(delta_kj - D_k.Pi_j),  w = diam^(2 - dim) |K^-1|_inf,
// which is Pi^T G Pi + w (I - D Pi)^T (I - D Pi) of MVEM.massHdiv entry by entry.  The entry q of cell_faces with
// i == 0 also tests the reference's assertion allclose(G, F D) and records the smallest failing cell in *bad.
template <int ND, class Out>
PB_HD void mvem_row(int64_t q, const DualTopo &T, const DualGeo &G, const Out &out, int32_t *bad) {
    const int64_t c = T.cf_cell[q];
    const int b = T.cf_ip[c], e = T.cf_ip[c + 1], i = (int)(q - b);
    double K[ND][ND], Ki[ND][ND], xc[ND];
    dual_perm<ND>(G, c, K);
    dual_inv<ND>(K, Ki);
    for (int k = 0; k < ND; ++k) xc[k] = G.ccent[k * G.nc + c];
    const double vol = G.vol[c], diam = dual_diameter(T, G, c);
    double knorm = 0.0;   // |K^-1|_inf, the largest absolute row sum
    for (int a = 0; a < ND; ++a) {
        double s = 0.0;
        for (int k = 0; k < ND; ++k) s += fabs(Ki[a][k]);
        knorm = s > knorm ? s : knorm;
    }
    double wpow = 1.0;    // diam^(2 - dim)
    if (ND == 1) wpow = diam;
    if (ND == 3) wpow = 1.0 / diam;
    const double w = wpow * knorm, gi = diam * diam / vol;   // G^-1 = gi K^-1

    // face j of the cell: F_j, D_j and Pi_j
    auto face = [&](int qj, double F[ND], double D[ND], double P[ND]) {
        const int32_t f = T.cf_ix[qj];
        const double s = (double)T.cf_sg[qj];
        for (int k = 0; k < ND; ++k) F[k] = s * (G.fcent[k * G.nf + f] - xc[k]) / diam;
        for (int k = 0; k < ND; ++k) {
            double t = 0.0;
            for (int m = 0; m < ND; ++m) t += G.fnorm[m * G.nf + f] * K[m][k];
            D[k] = t / diam;
        }
        for (int k = 0; k < ND; ++k) {
            double t = 0.0;
            for (int m = 0; m < ND; ++m) t += Ki[k][m] * F[m];
            P[k] = gi * t;
        }
    };
    if (i == 0) {   // mvem.py massHdiv: assert np.allclose(G, F @ D)
        double FD[ND][ND];
        for (int a = 0; a < ND; ++a)
            for (int k = 0; k < ND; ++k) FD[a][k] = 0.0;
        for (int qj = b; qj < e; ++qj) {
            double F[ND], D[ND], P[ND];
            face(qj, F, D, P);
            for (int a = 0; a < ND; ++a)
                for (int k = 0; k < ND; ++k) FD[a][k] += F[a] * D[k];
        }
        bool ok = true;
        for (int a = 0; a < ND; ++a)
            for (int k = 0; k < ND; ++k) {
                const double g = K[a][k] * vol / (diam * diam);
                ok = ok && fabs(g - FD[a][k]) <= 1e-8 + 1e-5 * fabs(FD[a][k]);
            }
        if (!ok) {
#ifdef __CUDA_ARCH__
            atomicMin(bad, (int32_t)c);
#else
            if (c < *bad) *bad = (int32_t)c;
#endif
        }
    }
    double Fi[ND], Di[ND], Pi[ND];
    face(b + i, Fi, Di, Pi);
    const int32_t fi = T.cf_ix[b + i];
    for (int qj = b; qj < e; ++qj) {
        double F[ND], D[ND], P[ND];
        face(qj, F, D, P);
        double cons = 0.0, stab = 0.0;
        for (int k = 0; k < ND; ++k) cons += Fi[k] * P[k];   // F_i^T G^-1 F_j
        // column i and j of I - D Pi, summed entry by entry: the expanded form cancels where the columns are small
        for (int qk = b; qk < e; ++qk) {
            double Fk[ND], Dk[ND], Pk[ND], ui = qk == b + i ? 1.0 : 0.0, uj = qk == qj ? 1.0 : 0.0;
            face(qk, Fk, Dk, Pk);
            for (int k = 0; k < ND; ++k) {
                ui -= Dk[k] * Pi[k];
                uj -= Dk[k] * P[k];
            }
            stab += ui * uj;
        }
        out.mvem_entry(T, fi, qj, cons, w, stab);
    }
    // vector_proj: R^T Pi(K = I) / diam = R^T s_i (x_i - x_c) / vol
    double p[ND];
    for (int k = 0; k < ND; ++k) p[k] = Fi[k] * diam / vol;
    out.template column<ND>(T, G, c, i, p);
}

// Node of the simplex c opposite its face at entry qi: a node of another face of c that face qi lacks.
template <int ND>
PB_HD int32_t rt0_opposite(const DualTopo &T, int64_t c, int qi) {
    const int32_t f = T.cf_ix[qi];
    const int qk = qi == T.cf_ip[c] ? qi + 1 : T.cf_ip[c];
    const int32_t g = T.cf_ix[qk];
    for (int r = T.fn_ip[g]; r < T.fn_ip[g + 1]; ++r) {
        const int32_t n = T.fn_ix[r];
        bool in = false;
        for (int s = T.fn_ip[f]; s < T.fn_ip[f + 1]; ++s) in = in || T.fn_ix[s] == n;
        if (!in) return n;
    }
    return T.fn_ix[T.fn_ip[g]];   // not reached on a simplex
}

// RT0 row: with x_a the vertices of the simplex, o_i the vertex opposite face i and s_i its sign,
//   A_ij = s_i s_j / (vol h) [ (sum_a (x_a - o_i))^T K^-1 (sum_b (x_b - o_j)) + sum_a (x_a - o_i)^T K^-1 (x_a - o_j) ],
// h = dim^2 (dim + 1)(dim + 2): C^T N^T HB (I (x) K^-1) / vol N C of RT0.massHdiv, since HB holds (1 + delta_ab) / h
// on the diagonal of every dim x dim block (a, b).  Flux reconstruction (faces_to_cell): R^T (x_c - o_i) /
// ((x_i - o_i) . n_i), x_i and n_i the centre and normal of face i.
template <int ND, class Out>
PB_HD void rt0_row(int64_t q, const DualTopo &T, const DualGeo &G, const Out &out) {
    const int64_t c = T.cf_cell[q];
    const int b = T.cf_ip[c], e = T.cf_ip[c + 1], i = (int)(q - b);
    double K[ND][ND], Ki[ND][ND];
    dual_perm<ND>(G, c, K);
    dual_inv<ND>(K, Ki);
    const double h = (double)(ND * ND * (ND + 1) * (ND + 2));
    auto node = [&](int32_t n, double x[ND]) {
        for (int k = 0; k < ND; ++k) x[k] = G.nodes[k * G.nn + n];
    };
    double oi[ND], si[ND];
    node(rt0_opposite<ND>(T, c, b + i), oi);
    for (int k = 0; k < ND; ++k) si[k] = 0.0;
    for (int qa = b; qa < e; ++qa) {
        double xa[ND];
        node(rt0_opposite<ND>(T, c, qa), xa);
        for (int k = 0; k < ND; ++k) si[k] += xa[k] - oi[k];
    }
    const double sgi = (double)T.cf_sg[b + i];
    const int32_t fi = T.cf_ix[b + i];
    for (int qj = b; qj < e; ++qj) {
        double oj[ND], sj[ND], KiSj[ND], acc = 0.0;
        node(rt0_opposite<ND>(T, c, qj), oj);
        for (int k = 0; k < ND; ++k) sj[k] = 0.0;
        for (int qa = b; qa < e; ++qa) {
            double xa[ND], v[ND];
            node(rt0_opposite<ND>(T, c, qa), xa);
            for (int k = 0; k < ND; ++k) {
                sj[k] += xa[k] - oj[k];
                v[k] = xa[k] - oj[k];
            }
            for (int k = 0; k < ND; ++k) {
                double t = 0.0;
                for (int m = 0; m < ND; ++m) t += Ki[k][m] * v[m];
                acc += (xa[k] - oi[k]) * t;
            }
        }
        for (int k = 0; k < ND; ++k) {
            double t = 0.0;
            for (int m = 0; m < ND; ++m) t += Ki[k][m] * sj[m];
            KiSj[k] = t;
        }
        for (int k = 0; k < ND; ++k) acc += si[k] * KiSj[k];
        const double a = sgi * (double)T.cf_sg[qj] * acc / (G.vol[c] * h);
        out.entry(T, fi, qj, a);
    }
    double den = 0.0, p[ND];
    for (int k = 0; k < ND; ++k) den += (G.fcent[k * G.nf + fi] - oi[k]) * G.fnorm[k * G.nf + fi];
    for (int k = 0; k < ND; ++k) p[k] = (G.ccent[k * G.nc + c] - oi[k]) / den;
    out.template column<ND>(T, G, c, i, p);
}

template <int ND>
PB_HD void dual_row(int method, int64_t q, const DualTopo &T, const DualGeo &G, double *mass, double *proj,
                    int32_t *bad) {
    const DualScatter out{mass, proj};
    if (method == kDualMvem) mvem_row<ND>(q, T, G, out, bad);
    else rt0_row<ND>(q, T, G, out);
}

}  // namespace pb
