// mpsa_node.cuh -- per-interaction-region MPSA-W (+ Biot coupling) assembly routine.
//
// Reference formulation (numerics/fv/mpsa.py:784-930): unknowns are the sub-cell displacement
// gradients G_K (order nd^2 * #subcells).  As for MPFA, displacement continuity at the
// continuity points, d_{K,f}.G_K[a,:] + u_{K,a} = ubar_{f,a}, holds exactly and each sub-cell has
// nd sub-faces at the node, so G_K[a,:] = D_K^{-1}(ubar_{F_K,a} - u_{K,a} 1): the unknowns that
// remain are the continuity-point displacements ubar_{f,a} (order nd * #subfaces: 36 instead
// of 72 on interior Cartesian nodes, 108 instead of 216 on 24-cell tetrahedral nodes).
//
//   traction functional of sub-cell K on sub-face f, component i (mpsa.py:1520-1675):
//     Tsym_{K,i}(n)  = sum_r n_r (C_K o S)[(i,r),:] vec(G_K)              own sub-cell
//     Tasym_i(n)     = sum_r n_r  SigmaA[(i,r)],
//     SigmaA[p]      = sum_{K'} w_{K'} (C_{K'} o !S)[p,:] vec(G_{K'})     node-volume average
//   rows: interior stress continuity (sym parts only, mpsa.py:884-892), Neumann / Robin
//   boundary rows incl. the asymmetric part unless eliminated (_eliminate_ncasym,
//   mpsa.py:1932-2000), Dirichlet rows ubar = u_b; right-hand sides: cell displacements,
//   boundary values (mpsa.py:984-1185) and, for Biot, the pressure jump n^T alpha
//   (biot.py:969-1019).  Outputs: hook (traction from the unique side, mpsa.py:1782-1832),
//   displacement trace (mpsa.py:760-781), and Biot's cell-row terms (biot.py:1054-1135).
#pragma once
#include "node_kernels.cuh"

namespace pb {

PB_HD int mpsa_width(int nd, int nsf, int nsc, int nb, int nalpha) {
    return (nsf * nd + nsc * nd + nb * nd + nalpha * nsc) | 1;
}
PB_HD int64_t mpsa_A_doubles(int nd, int nsf, int nsc, int nb, int nalpha) {
    return (int64_t)nsf * nd * mpsa_width(nd, nsf, nsc, nb, nalpha);
}
PB_HD int64_t mpsa_rest_doubles(int nd, int nsf, int nsc, int nb, int nalpha) {
    const int64_t nd2 = nd * nd, n = (int64_t)nsf * nd;
    const int64_t nrhs = (int64_t)nsc * nd + (int64_t)nb * nd + (int64_t)nalpha * nsc;
    int64_t d = (int64_t)nsc * nd2 * nd2;       // PS
    d += (int64_t)nsc * nd2;                    // E
    d += nd2 * (n + (int64_t)nsc * nd);         // SA | SAc
    d += nd2 * nrhs;                            // Z
    d += nsf;                                   // invmf
    d += (int64_t)nsf * nd;                     // nrm
    d += (int64_t)nsc;                          // volk
    d += (int64_t)nalpha * nsc * nd2 * 2;       // NA, AE
    int64_t ints = nsc + 4 * (int64_t)nsf + (int64_t)nsf * nd + n + (int64_t)nsc * nd + 2 * nd;
    return d + (ints + 1) / 2 + 2;
}

// 9-index of the stored (9,9,nc) stiffness for the local (i,r) pair (2-D: rows/cols
// 2,5,6,7,8 deleted, mpsa.py:1475-1480)
template <int ND>
PB_HD int c9(int i, int r) { return 3 * i + r; }

// symmetric-part mask S of _split_stiffness_matrix (mpsa.py:1461-1518) in local indices
template <int ND>
PB_HD bool sym_mask(int p, int q) {
    if (p == q) return true;
    // p = (i,i), q = (a,a), i != a  <->  (0,4),(0,8),(4,0),(4,8),(8,0),(8,4) in 3-D; (0,3),(3,0) in 2-D
    return (p % (ND + 1) == 0) && (q % (ND + 1) == 0);
}

template <int ND, class Solver, class Team>
PB_HD void mpsa_node(Team &t, const PlanView &P, const GeoView &G, const MpsaParams &prm,
                     const MpsaOut &o, int64_t s, double *pool, double *smd, double *scratch, int *err,
                     int64_t s_next = -1) {
    constexpr int ND2 = ND * ND;
    const int sc0 = P.node_sc_ptr[s], nsc = P.node_sc_ptr[s + 1] - sc0;
    const int sf0 = P.node_sf_ptr[s], nsf = P.node_sf_ptr[s + 1] - sf0;
    const int nb = P.node_nb[s];
    if (nsf == 0) return;
    const int nal = prm.n_alpha;
    const int n = nsf * ND;
    const int ncc = nsc * ND;        // cell-displacement columns
    const int nbc = nb * ND;         // boundary-value columns
    const int nrhs = ncc + nbc + nal * nsc;
    const int64_t nf = P.nf, nc = P.nc, nn = P.nn;

    double *PS = smd;                           // [k][p][a][m]
    double *E = PS + nsc * ND2 * ND2;           // [k][kappa][m]
    double *SA = E + nsc * ND2;                 // [p][x], x < n
    double *SAc = SA + ND2 * n;                 // [p][k*ND+a]
    double *Z = SAc + ND2 * ncc;                // [p][c], c < nrhs
    double *invmf = Z + ND2 * nrhs;
    double *nrm = invmf + nsf;                  // [u][r]  n_f / m_f
    double *volk = nrm + nsf * ND;
    double *NA = volk + nsc;                    // [q][k][m][i]  (n_{u(k,m)}^T alpha_k)_i
    double *AE = NA + nal * nsc * ND2;          // [q][k][a][m]  sum_kappa alpha_k[a][kappa] E_k[kappa][m]
    int *cell = (int *)(AE + nal * nsc * ND2);
    int *face = cell + nsc;
    int *sides = face + nsf;
    int *bloc = sides + nsf;
    int *bcu = bloc + nsf;                      // [u][i]
    int *rowidx = bcu + nsf * ND;
    int *slot = rowidx + n;
    int *elim = slot + nsc * ND;                // [i] neumann, [ND+i] robin
    int *sidesel = elim + 2 * ND;               // [u] side the traction is evaluated from

    // ---- phase 1: lists
    for (int k = t.tid(); k < nsc; k += t.size()) cell[k] = P.sc_cell[sc0 + k];
    for (int i = t.tid(); i < nsc * ND; i += t.size()) slot[i] = P.slot_sf[(int64_t)sc0 * ND + i];
    for (int u = t.tid(); u < nsf; u += t.size()) {
        const int64_t f = P.sf_face[sf0 + u];
        face[u] = (int)f;
        sides[u] = (int)P.sf_sides[sf0 + u];
        const int bl = P.sf_bloc[sf0 + u];
        bloc[u] = (bl == 0xFFFF) ? -1 : bl;
        const double im = 1.0 / (double)(P.fn_indptr[f + 1] - P.fn_indptr[f]);
        invmf[u] = im;
#pragma unroll
        for (int i = 0; i < ND; ++i) {
            int code = 0;
            if (bl != 0xFFFF) {
                code = prm.bc[i * nf + f];
                if (code == 0) code = 2;
            }
            bcu[u * ND + i] = code;
            nrm[u * ND + i] = G.fnorm[i * G.face_cs + f * G.face_es] * im;
        }
    }
    for (int x = t.tid(); x < n; x += t.size()) rowidx[x] = x;
    for (int i = t.tid(); i < ND2 * (n + ncc); i += t.size()) SA[i] = 0.0;
    t.sync();

    // ---- phase 2: per sub-cell  E = D^{-1}, weights, Biot helper products
    for (int k = t.tid(); k < nsc; k += t.size()) {
        const int64_t c = cell[k];
        double xc[ND], xs[ND], D[ND][ND], Ei[ND][ND];
#pragma unroll
        for (int i = 0; i < ND; ++i) {
            xc[i] = G.ccent[i * G.cell_cs + c * G.cell_es];
            xs[i] = G.nodes[i * G.node_cs + s * G.node_es];
        }
#pragma unroll
        for (int m = 0; m < ND; ++m) {
            const int u = slot[k * ND + m] >> 1;
            const int64_t f = face[u];
            const double e = (bloc[u] >= 0) ? 0.0 : prm.eta;
#pragma unroll
            for (int i = 0; i < ND; ++i) {
                const double xf = G.fcent[i * G.face_cs + f * G.face_es];
                D[m][i] = xf + e * (xs[i] - xf) - xc[i];
            }
        }
        if (!invert_small<ND>(D, Ei)) flag_singular(err, s);
#pragma unroll
        for (int q = 0; q < ND; ++q)
#pragma unroll
            for (int m = 0; m < ND; ++m) E[k * ND2 + q * ND + m] = Ei[q][m];
        volk[k] = G.cvol[c] / (double)P.sc_ncn[c];
        for (int q = 0; q < nal; ++q) {
            const double *al = prm.alpha + (int64_t)q * prm.alpha_stride;
            double a2[ND][ND];
#pragma unroll
            for (int a = 0; a < ND; ++a)
#pragma unroll
                for (int b = 0; b < ND; ++b) a2[a][b] = al[(3 * a + b) * prm.alpha_cs + c * prm.alpha_es];
#pragma unroll
            for (int m = 0; m < ND; ++m) {
                const int u = slot[k * ND + m] >> 1;
#pragma unroll
                for (int i = 0; i < ND; ++i) {
                    double v = 0.0, w = 0.0;
#pragma unroll
                    for (int r = 0; r < ND; ++r) {
                        v += nrm[u * ND + r] * a2[r][i];   // (n^T alpha)_i
                        w += a2[i][r] * Ei[r][m];          // AE[a=i][m]
                    }
                    NA[((q * nsc + k) * ND + m) * ND + i] = v;
                    AE[((q * nsc + k) * ND + i) * ND + m] = w;
                }
            }
        }
    }
    t.sync();
    // ---- phase 3: PS[k][p][a][m] = sum_kappa (C o S)[p,(a,kappa)] E[kappa][m];
    //               SA[p][(u,a)]  += w_k sum_kappa (C o !S)[p,(a,kappa)] E[kappa][m]
    for (int it = t.tid(); it < nsc * ND2; it += t.size()) {
        const int k = it / ND2, p = it - k * ND2;
        const int64_t c = cell[k];
        const int pi = p / ND, pr = p - pi * ND;
        const double *Crow = prm.stiff + (int64_t)c9<ND>(pi, pr) * 9 * prm.stiff_cs + c * prm.stiff_es;  // C[p9][q9][c]
#pragma unroll
        for (int a = 0; a < ND; ++a) {
            double cs[ND];
#pragma unroll
            for (int q = 0; q < ND; ++q)
                cs[q] = sym_mask<ND>(p, a * ND + q) ? Crow[(int64_t)c9<ND>(a, q) * prm.stiff_cs] : 0.0;
#pragma unroll
            for (int m = 0; m < ND; ++m) {
                double v = 0.0;
#pragma unroll
                for (int q = 0; q < ND; ++q) v += cs[q] * E[k * ND2 + q * ND + m];
                PS[((k * ND2 + p) * ND + a) * ND + m] = v;
            }
        }
    }
    // one item per (p, a, sub-cell); a sub-face entry of SigmaA receives one contribution per side
    // (<= 2, so the sum does not depend on the order).  Node-volume weights w_K = vol_K / sum vol
    // (mpsa.py:1619-1640) are formed on the fly.
    for (int it = t.tid(); it < ND2 * ND * nsc; it += t.size()) {
        const int pa = it / nsc, k = it - pa * nsc;
        const int p = pa / ND, a = pa - p * ND;
        const int pi = p / ND, pr = p - pi * ND;
        double tot = 0.0;
        for (int j = 0; j < nsc; ++j) tot += volk[j];
        const double w = volk[k] / tot;
        const int64_t c = cell[k];
        const double *Crow = prm.stiff + (int64_t)c9<ND>(pi, pr) * 9 * prm.stiff_cs + c * prm.stiff_es;
        double ca[ND];
#pragma unroll
        for (int q = 0; q < ND; ++q)
            ca[q] = sym_mask<ND>(p, a * ND + q) ? 0.0 : w * Crow[(int64_t)c9<ND>(a, q) * prm.stiff_cs];
        double sum = 0.0;
#pragma unroll
        for (int m = 0; m < ND; ++m) {
            double v = 0.0;
#pragma unroll
            for (int q = 0; q < ND; ++q) v += ca[q] * E[k * ND2 + q * ND + m];
            team_add(SA + p * n + (slot[k * ND + m] >> 1) * ND + a, v);
            sum += v;
        }
        SAc[p * ncc + k * ND + a] = -sum;
    }
    // elimination flags of _eliminate_ncasym (mpsa.py:1932-2000), one thread per component
    for (int i = t.tid(); i < ND; i += t.size()) {
        int cn = 0, cr = 0;
        for (int u = 0; u < nsf; ++u) {
            cn += bcu[u * ND + i] == 2;
            cr += bcu[u * ND + i] == 3;
        }
        elim[i] = nsc < cn;
        elim[ND + i] = nsc < cr;
    }
    t.sync();

    // ---- phase 3b: side each sub-face's traction is evaluated from.  The reference takes the
    // side with the smaller cell index (mpsa.py:1782-1832); traction continuity makes both sides
    // agree, and the softer side is the well-conditioned one in the continuity-point formulation
    // (see the MPFA routine), so pick the side with the smaller |n . (C o S) D^-1|.
    for (int u = t.tid(); u < nsf; u += t.size()) {
        const int s1 = sides[u] & 0xFFFF, s2 = (sides[u] >> 16) & 0xFFFF;
        int pick = s1;
        if (s2 != 0xFFFF) {
            const double *nu = nrm + u * ND;
            double w1 = 0.0, w2 = 0.0;
            const double *p1 = PS + (s1 / ND) * ND2 * ND2, *p2 = PS + (s2 / ND) * ND2 * ND2;
            for (int i = 0; i < ND; ++i)
                for (int am = 0; am < ND2; ++am) {
                    double a1 = 0.0, a2 = 0.0;
#pragma unroll
                    for (int r = 0; r < ND; ++r) {
                        a1 += nu[r] * p1[(i * ND + r) * ND2 + am];
                        a2 += nu[r] * p2[(i * ND + r) * ND2 + am];
                    }
                    w1 += fabs(a1);
                    w2 += fabs(a2);
                }
            if (w2 < w1) pick = s2;
        }
        sidesel[u] = pick;
    }
    t.sync();

    // ---- phase 4: row x = (sub-face, component) of the local system, handed to the solver row by row (the solver
    // scales it to unit 1-norm, matrix_operations.py:1880-1906)
    auto row_of = [&](int x, double *row) {
        const int u = x / ND, i = x - u * ND;
        const int code = bcu[x];
        if (code == 1 && prm.basis == nullptr) {  // Dirichlet component: ubar_{u,i} = u_b
            row[x] = 1.0;
            row[n + ncc + bloc[u] * ND + i] = 1.0;
            return;
        }
        const double *nu = nrm + u * ND;
        if (prm.basis != nullptr && bloc[u] >= 0) {
            // Boundary conditions given in a rotated basis B_f (bc.basis; _fvutils.py:765-945): the nd
            // equations of the sub-face are multiplied by B_f before the per-component exclusion, the
            // boundary values live in the rotated frame.  Row i = sum_j B[i][j] (equation j).
            const int64_t fb = face[u];
            double B[ND][ND];
#pragma unroll
            for (int a = 0; a < ND; ++a)
#pragma unroll
                for (int j = 0; j < ND; ++j) B[a][j] = prm.basis[(int64_t)(a * ND + j) * nf + fb];
            if (code == 1) {
#pragma unroll
                for (int j = 0; j < ND; ++j) row[u * ND + j] = B[i][j];
                row[n + ncc + bloc[u] * ND + i] = 1.0;
            } else {
                const int side = sides[u] & 0xFFFF;  // boundary sub-face: one side
                const int k = side / ND;
                const double sg = (slot[side] & 1) ? -1.0 : 1.0;
                for (int j = 0; j < ND; ++j) {
                    const double wgt = sg * B[i][j];
                    if (wgt == 0.0) continue;
                    const double *ps = PS + (k * ND2 + j * ND) * ND2;  // [r][a][m], traction component j
#pragma unroll
                    for (int a = 0; a < ND; ++a) {
                        double csum = 0.0;
#pragma unroll
                        for (int m = 0; m < ND; ++m) {
                            double v = 0.0;
#pragma unroll
                            for (int r = 0; r < ND; ++r) v += nu[r] * ps[(r * ND + a) * ND + m];
                            v *= wgt;
                            row[(slot[k * ND + m] >> 1) * ND + a] += v;
                            csum += v;
                        }
                        row[n + k * ND + a] += csum;
                    }
                    for (int q = 0; q < nal; ++q)
                        row[n + ncc + nbc + q * nsc + k] += wgt * NA[((q * nsc + k) * ND + (side - k * ND)) * ND + j];
                    // asymmetric part of component j unless eliminated for (its flag, j) (mpsa.py:1932-2000)
                    const int cj = bcu[u * ND + j];
                    if (!((cj == 2 && elim[j]) || (cj == 3 && elim[ND + j]))) {
                        for (int c = 0; c < n; ++c) {
                            double v = 0.0;
#pragma unroll
                            for (int r = 0; r < ND; ++r) v += nu[r] * SA[(j * ND + r) * n + c];
                            row[c] += wgt * v;
                        }
                        for (int c = 0; c < ncc; ++c) {
                            double v = 0.0;
#pragma unroll
                            for (int r = 0; r < ND; ++r) v += nu[r] * SAc[(j * ND + r) * ncc + c];
                            row[n + c] -= wgt * v;
                        }
                    }
                }
                row[n + ncc + bloc[u] * ND + i] = invmf[u];
                if (code == 3) {  // Robin weight acts on the rotated displacement: w B ubar
                    const double as = G.farea[fb] * invmf[u];
#pragma unroll
                    for (int j = 0; j < ND; ++j) {
                        double wb = 0.0;
#pragma unroll
                        for (int kk = 0; kk < ND; ++kk)
                            wb += (prm.robw ? prm.robw[(int64_t)(i * ND + kk) * nf + fb] : (i == kk ? 1.0 : 0.0)) * B[kk][j];
                        row[u * ND + j] += as * wb;
                    }
                }
            }
            return;
        }
        for (int sd = 0; sd < 2; ++sd) {
            const int side = sd == 0 ? (sides[u] & 0xFFFF) : ((sides[u] >> 16) & 0xFFFF);
            if (side == 0xFFFF) continue;
            const int k = side / ND;
            const double sg = (slot[side] & 1) ? -1.0 : 1.0;
            const double *ps = PS + (k * ND2 + i * ND) * ND2;  // [r][a][m]
#pragma unroll
            for (int a = 0; a < ND; ++a) {
                double csum = 0.0;
#pragma unroll
                for (int m = 0; m < ND; ++m) {
                    double v = 0.0;
#pragma unroll
                    for (int r = 0; r < ND; ++r) v += nu[r] * ps[(r * ND + a) * ND + m];
                    v *= sg;
                    row[(slot[k * ND + m] >> 1) * ND + a] += v;
                    csum += v;
                }
                row[n + k * ND + a] += csum;
            }
            for (int q = 0; q < nal; ++q)  // Biot pressure jump (biot.py:969-1019)
                row[n + ncc + nbc + q * nsc + k] += sg * NA[((q * nsc + k) * ND + (side - k * ND)) * ND + i];
            if (code != 0) {  // boundary Neumann / Robin row: asymmetric part (single side)
                const bool el = code == 2 ? elim[i] : elim[ND + i];
                if (!el) {
                    for (int c = 0; c < n; ++c) {
                        double v = 0.0;
#pragma unroll
                        for (int r = 0; r < ND; ++r) v += nu[r] * SA[(i * ND + r) * n + c];
                        row[c] += sg * v;
                    }
                    for (int c = 0; c < ncc; ++c) {
                        double v = 0.0;
#pragma unroll
                        for (int r = 0; r < ND; ++r) v += nu[r] * SAc[(i * ND + r) * ncc + c];
                        row[n + c] -= sg * v;
                    }
                }
            }
        }
        if (code == 2 || code == 3) row[n + ncc + bloc[u] * ND + i] = invmf[u];  // mpsa.py:1123-1137
        if (code == 3) {  // Robin: + (A_f/m_f) sum_j w[i][j] ubar_{u,j}  (mpsa.py:1381-1459)
            const int64_t f = face[u];
            const double as = G.farea[f] * invmf[u];
#pragma unroll
            for (int j = 0; j < ND; ++j) {
                const double w = prm.robw ? prm.robw[(int64_t)(i * ND + j) * nf + f] : (i == j ? 1.0 : 0.0);
                row[u * ND + j] += as * w;
            }
        }
    };

    // ---- phase 5: solve; X[rowidx[x]*ldx + c] is the solution
    const double *X;
    int ldx;
    if (!Solver::solve_rows(t, row_of, n, nrhs, pool, rowidx, scratch, X, ldx)) {
        if (t.tid() == 0) flag_singular(err, s);
        t.sync();
        return;
    }

#if defined(__CUDA_ARCH__)
    // software prefetch of the NEXT region's inputs into L2 (three dependent stages spread over
    // phases 6-7 so that no stage waits): pointers here, lists after phase 6, records after phase 7
    int pf_sc0 = 0, pf_nsc = 0, pf_sf0 = 0, pf_nsf = 0;
    int64_t pf_pos0 = 0;
    if (s_next >= 0) {
        pf_sc0 = P.node_sc_ptr[s_next];
        pf_nsc = P.node_sc_ptr[s_next + 1] - pf_sc0;
        pf_sf0 = P.node_sf_ptr[s_next];
        pf_nsf = P.node_sf_ptr[s_next + 1] - pf_sf0;
        pf_pos0 = P.posfc_ptr[s_next];
    }
#endif
    // ---- phase 6: Z[p][c] = SigmaA[p] applied to the solution (+ direct cell-displacement term)
#if defined(__CUDA_ARCH__)
    // (ND2 x n) * (n x nrhs) on the FP64 tensor cores: one 16x8 tile of Z per warp iteration (m16n8k4)
    {
        const int l = t.lane();
        const int ntr = (ND2 + 15) / 16, ntc = (nrhs + 7) / 8;
        for (int tile = t.warp(); tile < ntr * ntc; tile += t.nwarps()) {
            const int tr = tile / ntc, tc = tile - tr * ntc;
            const int row0 = 16 * tr + (l >> 2), row1 = row0 + 8;
            const int colb = 8 * tc + (l >> 2);
            double acc0[2] = {0.0, 0.0}, acc1[2] = {0.0, 0.0};
            for (int k0 = 0; k0 < n; k0 += 4) {
                const int k = k0 + (l & 3);
                const double a0 = (row0 < ND2 && k < n) ? SA[row0 * n + k] : 0.0;
                const double a1 = (row1 < ND2 && k < n) ? SA[row1 * n + k] : 0.0;
                const double b = (k < n && colb < nrhs) ? X[rowidx[k] * ldx + colb] : 0.0;
                pb_dmma2(acc0, acc1, a0, a1, b);
            }
            const int c0 = 8 * tc + 2 * (l & 3);
            const int rows[2] = {row0, row1};
            const double *accs[2] = {acc0, acc1};
            for (int h = 0; h < 2; ++h) {
                const int row = rows[h];
                if (row < ND2) {
                    if (c0 < nrhs) Z[row * nrhs + c0] = accs[h][0] + (c0 < ncc ? SAc[row * ncc + c0] : 0.0);
                    if (c0 + 1 < nrhs)
                        Z[row * nrhs + c0 + 1] = accs[h][1] + (c0 + 1 < ncc ? SAc[row * ncc + c0 + 1] : 0.0);
                }
            }
        }
    }
#else
    for (int it = t.tid(); it < ND2 * nrhs; it += t.size()) {
        const int p = it / nrhs, c = it - p * nrhs;
        double v = (c < ncc) ? SAc[p * ncc + c] : 0.0;
        for (int x = 0; x < n; ++x) v += SA[p * n + x] * X[(int64_t)rowidx[x] * ldx + c];
        Z[it] = v;
    }
#endif
    t.sync();

#if defined(__CUDA_ARCH__)
    int pf_cell = -1, pf_face = -1;
    if (t.tid() < pf_nsc) pf_cell = P.sc_cell[pf_sc0 + t.tid()];
    if (t.tid() < pf_nsf) {
        pf_face = P.sf_face[pf_sf0 + t.tid()];
        if ((t.tid() & 7) == 0) {
            pb_prefetch_l2(P.sf_sides + pf_sf0 + t.tid());
            pb_prefetch_l2(P.sf_bloc + pf_sf0 + t.tid());
        }
    }
    if (t.tid() * 16 < pf_nsc * ND) pb_prefetch_l2(P.slot_sf + (int64_t)pf_sc0 * ND + t.tid() * 16);
    for (int64_t off = (int64_t)t.tid() * 32; off < (int64_t)pf_nsf * pf_nsc; off += (int64_t)t.size() * 32)
        pb_prefetch_l2(P.pos_fc + pf_pos0 + off);
#endif
    // ---- phase 7: face rows (traction from the unique side, displacement trace)
    const int32_t *pfc = P.pos_fc + P.posfc_ptr[s];
    const int32_t *pfb = P.pos_fb + P.posfb_ptr[s];
    // one warp per sub-face, lanes over the right-hand-side columns, the nd components of the
    // row inside: the 9 solution rows of the selected sub-cell and the CSR position are loaded
    // once per (sub-face, column) instead of once per component
    for (int u = t.warp(); u < nsf; u += t.nwarps()) {
        const double *nu = nrm + u * ND;
        const int side1 = sidesel[u];
        const int k1 = side1 / ND, m1 = side1 - k1 * ND;
        double hs[ND][ND][ND];  // [i][a][m] coefficient of ubar_{u(k1,m),a} in component i
        double hsum[ND][ND];    // [i][a] = sum_m hs[i][a][m]
#pragma unroll
        for (int i = 0; i < ND; ++i) {
            const double *ps1 = PS + (k1 * ND2 + i * ND) * ND2;
#pragma unroll
            for (int a = 0; a < ND; ++a) {
                double sm = 0.0;
#pragma unroll
                for (int m = 0; m < ND; ++m) {
                    double v = 0.0;
#pragma unroll
                    for (int r = 0; r < ND; ++r) v += nu[r] * ps1[(r * ND + a) * ND + m];
                    hs[i][a][m] = v;
                    sm += v;
                }
                hsum[i][a] = sm;
            }
        }
        int xo[ND][ND];  // offsets of the solution rows of ubar_{u(k1,m),a}
#pragma unroll
        for (int a = 0; a < ND; ++a)
#pragma unroll
            for (int m = 0; m < ND; ++m) xo[a][m] = rowidx[(slot[k1 * ND + m] >> 1) * ND + a] * ldx;
        bool use_asym[ND];
        int uo[ND];
#pragma unroll
        for (int i = 0; i < ND; ++i) {
            const int code = bcu[u * ND + i];
            use_asym[i] = !((code == 2 && elim[i]) || (code == 3 && elim[ND + i]));
            uo[i] = rowidx[u * ND + i] * ldx;
        }
        const double im = invmf[u];
        const int64_t f = face[u];
        const int64_t fc0 = P.fc_indptr[f], fcl = P.fc_indptr[f + 1] - fc0;
        const int64_t fb0 = P.fb_indptr[f], fbl = P.fb_indptr[f + 1] - fb0;
        for (int c = t.lane(); c < nrhs; c += t.lanes()) {
            double hk[ND], tr[ND];
#pragma unroll
            for (int i = 0; i < ND; ++i) hk[i] = 0.0;
#pragma unroll
            for (int a = 0; a < ND; ++a)
#pragma unroll
                for (int m = 0; m < ND; ++m) {
                    const double xv = X[xo[a][m] + c];
#pragma unroll
                    for (int i = 0; i < ND; ++i) hk[i] += hs[i][a][m] * xv;
                }
#pragma unroll
            for (int i = 0; i < ND; ++i) {
                if (use_asym[i]) {
#pragma unroll
                    for (int r = 0; r < ND; ++r) hk[i] += nu[r] * Z[(i * ND + r) * nrhs + c];
                }
                tr[i] = X[uo[i] + c] * im;
            }
            if (c < ncc) {
                const int k = c / ND, j = c - k * ND;
                if (k == k1) {  // direct dependence of the own sub-cell's gradient on u_{k1,j}
#pragma unroll
                    for (int i = 0; i < ND; ++i) {
                        double hj = hsum[i][0];
#pragma unroll
                        for (int a = 1; a < ND; ++a) hj = (j == a) ? hsum[i][a] : hj;
                        hk[i] -= hj;
                    }
                }
                const int64_t pb = pfc[u * nsc + k];
                const int64_t pos = ND2 * fc0 + (pb - fc0) * ND + j;
#pragma unroll
                for (int i = 0; i < ND; ++i) {
                    if (o.stress) red_add(o.stress + pos + (int64_t)i * ND * fcl, hk[i]);
                    if (o.bdc) red_add(o.bdc + pos + (int64_t)i * ND * fcl, tr[i]);
                }
            } else if (c < ncc + nbc) {
                const int cb = c - ncc;
                const int b = cb / ND, j = cb - b * ND;
                const int64_t pb = pfb[u * nb + b];
                const int64_t pos = ND2 * fb0 + (pb - fb0) * ND + j;
#pragma unroll
                for (int i = 0; i < ND; ++i) {
                    if (o.bstress) red_add(o.bstress + pos + (int64_t)i * ND * fbl, hk[i]);
                    if (o.bdf) red_add(o.bdf + pos + (int64_t)i * ND * fbl, tr[i]);
                }
            } else {
                const int cq = c - ncc - nbc;
                const int q = cq / nsc, k = cq - q * nsc;
                const int64_t pb = pfc[u * nsc + k];
                const int64_t pos = ND * fc0 + (pb - fc0);
#pragma unroll
                for (int i = 0; i < ND; ++i) {
                    double h = hk[i];
                    if (k == k1) h -= NA[((q * nsc + k1) * ND + m1) * ND + i];  // biot.py:853-855
                    if (o.sg[q]) red_add(o.sg[q] + pos + (int64_t)i * fcl, h);
                    if (o.bdp[q]) red_add(o.bdp[q] + pos + (int64_t)i * fcl, tr[i]);
                }
            }
        }
    }
#if defined(__CUDA_ARCH__)
    if (pf_cell >= 0) {
        if (prm.stiff_cs == 1) {
            const double *rec = prm.stiff + (int64_t)pf_cell * prm.stiff_es;
#pragma unroll
            for (int b = 0; b < 81; b += 16) pb_prefetch_l2(rec + b);
            pb_prefetch_l2(rec + 80);
        }
        if (G.cell_cs == 1) pb_prefetch_l2(G.ccent + (int64_t)pf_cell * G.cell_es);
        pb_prefetch_l2(G.cvol + pf_cell);
        pb_prefetch_l2(P.sc_ncn + pf_cell);
    }
    if (pf_face >= 0) {
        if (G.face_cs == 1) {
            pb_prefetch_l2(G.fnorm + (int64_t)pf_face * G.face_es);
            pb_prefetch_l2(G.fcent + (int64_t)pf_face * G.face_es);
        }
        pb_prefetch_l2(P.fn_indptr + pf_face);
        pb_prefetch_l2(P.fc_indptr + pf_face);
#pragma unroll
        for (int i = 0; i < ND; ++i) pb_prefetch_l2(prm.bc + (int64_t)i * nf + pf_face);
    }
#endif
    // ---- phase 8 (Biot): cell rows  dv_K . G_K  (biot.py:1054-1135)
    if (nal > 0) {
        const int32_t *pcc = P.pos_cc + P.poscc_ptr[s];
        const int32_t *pcb = P.pos_cb + P.poscb_ptr[s];
        for (int it = t.warp(); it < nal * nsc; it += t.nwarps()) {
            const int q = it / nsc, k = it - q * nsc;
            const double *ae = AE + (q * nsc + k) * ND2;  // [a][m]
            const double vol = volk[k];
            const double *xr[ND][ND];
#pragma unroll
            for (int a = 0; a < ND; ++a)
#pragma unroll
                for (int m = 0; m < ND; ++m)
                    xr[a][m] = X + (int64_t)rowidx[(slot[k * ND + m] >> 1) * ND + a] * ldx;
            for (int c = t.lane(); c < nrhs; c += t.lanes()) {
                double v = 0.0;
#pragma unroll
                for (int a = 0; a < ND; ++a)
#pragma unroll
                    for (int m = 0; m < ND; ++m) v += ae[a * ND + m] * xr[a][m][c];
                if (c < ncc) {
                    const int k2 = c / ND, j = c - k2 * ND;
                    if (k2 == k) {
#pragma unroll
                        for (int m = 0; m < ND; ++m) v -= ae[j * ND + m];
                    }
                    if (o.dd[q]) red_add(o.dd[q] + (int64_t)pcc[k * nsc + k2] * ND + j, vol * v);
                } else if (c < ncc + nbc) {
                    const int cb = c - ncc;
                    const int b = cb / ND, j = cb - b * ND;
                    if (o.bdd[q]) red_add(o.bdd[q] + (int64_t)pcb[k * nb + b] * ND + j, vol * v);
                } else {
                    const int cq = c - ncc - nbc;
                    const int q2 = cq / nsc, k2 = cq - q2 * nsc;
                    if (q2 == q && o.cons[q]) red_add(o.cons[q] + (int64_t)pcc[k * nsc + k2], vol * v);
                }
            }
        }
    }
    t.sync();
}

}  // namespace pb
