"""Extended-precision restatement of the mixed schemes' local matrices (csrc/dual_cell.cuh: MVEM.massHdiv of
numerics/vem/mvem.py, RT0.massHdiv of numerics/fem/rt0.py) and of their hybridization (csrc/dual_hybrid.cuh:
HybridDualVEM.matrix_rhs of numerics/vem/hybrid.py), in mpmath at 40 digits from the very float64 arrays the kernels
receive: the geometry in the grid's frame, the tensor, the rotation, the aperture.  Every value comes with its own
error scale, built from the cells it sums over, so that a check at a fixed multiple of the scale is as tight on the
cells of permeability 1 as on those of permeability 10^6:

  mass entry (f, g):    sum over the cells of f and g of max |A_c|, A_c the cell's local matrix;
  face-system entry:    sum over the cells of the entry of kappa(A_c) max |E_c|, E_c = A_c^-1 and kappa the 2-norm
                        condition number (the inverse loses kappa rounding errors of its own size);
  right-hand side, p, u: kappa times the first-order sum of what the value's errors in E, z and S bring in.

Test infrastructure only."""
from __future__ import annotations

import numpy as np
import scipy.sparse as sps
from mpmath import mp

DPS = 40

# Bounds, in units of the scales above.
# MASS_TOL: an MVEM entry sums n consistency and n^2 stabilization products of inputs rounded once each, RT0 a few
#   dozen; the host build stays within 1.6e-14 on every fixture and polygon (RT0 on the structured tetrahedra, MVEM on
#   the perturbed hexahedra), so 1e-13 leaves a factor six for the device's fused multiply-adds.  A relative change of
#   1e-9 in one cell's matrix is four orders of magnitude above it.
# PROJ_TOL: a column of the flux reconstruction is one difference and one quotient per component; 4e-16 measured.
# HYBRID_TOL: Gauss-Jordan inverts an n x n matrix to a backward error of about n eps, i.e. 3.6e-15 kappa |E| at the
#   32 faces of one warp; the host build stays within 1.5e-16 of the scales, so 1e-14 bounds the device too.
MASS_TOL, PROJ_TOL, HYBRID_TOL = 1e-13, 1e-14, 1e-14


class Topo:
    """cell_faces with the faces of every cell sorted (as the kernels read it), face_nodes, and the first (smallest)
    cell of every face."""

    def __init__(self, g):
        cf = sps.csc_matrix(g.cell_faces, copy=True)
        cf.sort_indices()
        fn = sps.csc_matrix(g.face_nodes)
        self.nd, self.nc, self.nf = int(g.dim), g.num_cells, g.num_faces
        self.ip, self.ix, self.sg = cf.indptr, cf.indices, np.asarray(cf.data).astype(int)
        self.fn_ip, self.fn_ix = fn.indptr, fn.indices
        self.first = np.full(self.nf, np.iinfo(np.int64).max)
        for c in range(self.nc - 1, -1, -1):
            self.first[self.faces(c)] = c

    def faces(self, c):
        return self.ix[self.ip[c]:self.ip[c + 1]]

    def signs(self, c):
        return self.sg[self.ip[c]:self.ip[c + 1]]

    def cell_nodes(self, c):
        return np.unique(np.concatenate([self.fn_ix[self.fn_ip[f]:self.fn_ip[f + 1]] for f in self.faces(c)]))


def _m(a):
    return mp.matrix([[mp.mpf(float(x)) for x in row] for row in np.atleast_2d(a)])


def _f(M):
    return np.array([[float(M[i, j]) for j in range(M.cols)] for i in range(M.rows)])


def mvem_cell(T, c, geo, perm, inv_a=1.0):
    """MVEM's local matrix of cell c, Pi^T G Pi / a + w (I - D Pi)^T (I - D Pi) (mvem.py massHdiv; the aperture a
    scales the volume and the normals, hybrid.py), and the flux reconstruction s_i (x_i - x_c) / vol of its faces in
    the frame (n x nd)."""
    nodes, fnorm, fcent, ccent, vol = geo[:5]
    nd, f, s = T.nd, T.faces(c), [int(v) for v in T.signs(c)]
    n = f.size
    x = [[mp.mpf(float(v)) for v in nodes[k, T.cell_nodes(c)]] for k in range(3)]
    m = len(x[0])
    d2 = max(sum((x[k][a] - x[k][b]) ** 2 for k in range(3)) for a in range(m) for b in range(a, m))
    diam = mp.sqrt(d2)
    K = _m(perm[:nd, :nd, c])
    Ki = K ** -1
    knorm = max(sum(abs(Ki[a, k]) for k in range(nd)) for a in range(nd))
    w = diam ** (2 - nd) * knorm
    xc = [mp.mpf(float(ccent[k, c])) for k in range(nd)]
    vc = mp.mpf(float(vol[c]))
    F, N = mp.matrix(nd, n), mp.matrix(nd, n)
    for j in range(n):
        for k in range(nd):
            F[k, j] = s[j] * (mp.mpf(float(fcent[k, f[j]])) - xc[k]) / diam
            N[k, j] = mp.mpf(float(fnorm[k, f[j]]))
    D = K.T * N / diam
    Pi = Ki * F * (diam ** 2 / vc)                  # G^-1 F, G = K vol / diam^2
    IP = mp.eye(n) - D.T * Pi
    A = (F.T * Pi) * mp.mpf(float(inv_a)) + w * (IP.T * IP)    # inv_a = 1 / a as the kernel receives it
    proj = [[s[i] * (mp.mpf(float(fcent[k, f[i]])) - xc[k]) / vc for k in range(nd)] for i in range(n)]
    return A, proj


def rt0_cell(T, c, geo, perm):
    """RT0's local matrix of the simplex c in closed form (dual_cell.cuh rt0_row, rt0.py massHdiv) and its flux
    reconstruction (x_c - o_i) / ((x_i - o_i) . n_i), o_i the vertex opposite face i."""
    nodes, fnorm, fcent, ccent, vol = geo[:5]
    nd, f, s = T.nd, T.faces(c), [int(v) for v in T.signs(c)]
    n = f.size
    cn = T.cell_nodes(c)
    opp = [int(np.setdiff1d(cn, T.fn_ix[T.fn_ip[fi]:T.fn_ip[fi + 1]])[0]) for fi in f]
    X = [[mp.mpf(float(nodes[k, o])) for k in range(nd)] for o in opp]
    Ki = _m(perm[:nd, :nd, c]) ** -1
    h = nd * nd * (nd + 1) * (nd + 2)
    vc = mp.mpf(float(vol[c]))

    def q(u, v):
        return sum(u[k] * Ki[k, m] * v[m] for k in range(nd) for m in range(nd))

    A = mp.matrix(n, n)
    for i in range(n):
        si = [sum(X[a][k] - X[i][k] for a in range(n)) for k in range(nd)]
        for j in range(n):
            sj = [sum(X[a][k] - X[j][k] for a in range(n)) for k in range(nd)]
            acc = q(si, sj) + sum(q([X[a][k] - X[i][k] for k in range(nd)], [X[a][k] - X[j][k] for k in range(nd)])
                                  for a in range(n))
            A[i, j] = s[i] * s[j] * acc / (vc * h)
    proj = []
    for i in range(n):
        den = sum((mp.mpf(float(fcent[k, f[i]])) - X[i][k]) * mp.mpf(float(fnorm[k, f[i]])) for k in range(nd))
        proj.append([(mp.mpf(float(ccent[k, c])) - X[i][k]) / den for k in range(nd)])
    return A, proj


def mass_reference(g, method, geo, perm, rot):
    """The global mass matrix (dense, nf x nf) and the flux reconstruction values (in the layout of
    ``DualGrid.download``: 3 cf_ip[c] + a n + i), each with its per-entry scale."""
    T = Topo(g)
    M, Ms = np.zeros((T.nf, T.nf)), np.zeros((T.nf, T.nf))
    P, Ps = np.zeros(3 * T.ip[-1]), np.zeros(3 * T.ip[-1])
    R = _m(rot)
    with mp.workdps(DPS):
        for c in range(T.nc):
            A, proj = (mvem_cell if method == 0 else rt0_cell)(T, c, geo, perm)
            Af = _f(A)
            f = T.faces(c)
            M[np.ix_(f, f)] += Af
            Ms[np.ix_(f, f)] += np.abs(Af).max()
            b, n = T.ip[c], f.size
            amb = [[float(sum(R[k, a] * proj[i][k] for k in range(T.nd))) for a in range(3)] for i in range(n)]
            sc = max(abs(float(v)) for row in proj for v in row)
            for i in range(n):
                for a in range(3):
                    P[3 * b + a * n + i] = amb[i][a]
                    Ps[3 * b + a * n + i] = sc
    return M, Ms, P, Ps


class HybridReference:
    """The condensation of every cell (VEM mode, r = 0, h = -source): E = A^-1, z = -E 1, t = 1^T E 1, S = 1 / t,
    L = z S z^T - E, the face matrix H with hybrid.py's boundary rows and its right-hand side, each with its scale;
    ``recover`` restates p = S (-z^T lambda - h) and u_f = s_i (E (p 1 - lambda))_i from the face's first cell."""

    def __init__(self, g, geo, codes, values):
        T = self.T = Topo(g)
        nf, nc = T.nf, T.nc
        areas = np.asarray(g.face_areas, float)
        self.cells = []
        H, Hs = np.zeros((nf, nf)), np.zeros((nf, nf))
        rhs, rs = np.zeros(nf), np.zeros(nf)
        perm, aper = geo[5], geo[7]
        with mp.workdps(DPS):
            for c in range(nc):
                A, _ = mvem_cell(T, c, geo, perm, 1.0 / float(aper[c]))
                s = [int(v) for v in T.signs(c)]
                n = len(s)
                for i in range(n):
                    for j in range(n):
                        A[i, j] *= s[i] * s[j]
                E = A ** -1
                z = [-sum(E[i, j] for j in range(n)) for i in range(n)]
                t = -sum(z)
                S = 1 / t
                h = -mp.mpf(float(values[nf + c]))
                L = mp.matrix(n, n)
                for i in range(n):
                    for j in range(n):
                        L[i, j] = z[i] * S * z[j] - E[i, j]
                Ef = _f(E)
                kappa = np.linalg.cond(_f(A))
                f = T.faces(c)
                H[np.ix_(f, f)] += _f(L)
                Hs[np.ix_(f, f)] += kappa * np.abs(Ef).max()
                term = np.array([float(-S * z[i] * h) for i in range(n)])
                rhs[f] += term
                # first order in the errors of E: those of z_i (row i of E) and of S (all of E)
                rho, Sf, zf = np.abs(Ef).sum(axis=1), abs(float(S)), np.abs(_f(mp.matrix(z)).ravel())
                rs[f] += kappa * Sf * abs(float(h)) * (rho + Sf * zf * rho.sum())
                self.cells.append((E, z, t, h, Ef, kappa))
        norm = np.abs(H).sum(axis=1).max()
        norm_scale = Hs.sum(axis=1).max()
        bc = np.asarray(values[:nf], float)
        sign = np.array([T.signs(T.first[f])[np.searchsorted(T.faces(T.first[f]), f)] for f in range(nf)])
        for f in range(nf):
            if codes[f] == 1:      # PB_BC_DIR: row cleared, |H|_inf on the diagonal, rhs |H|_inf bc
                H[f], Hs[f] = 0.0, 0.0
                H[f, f], Hs[f, f] = norm, norm_scale
                rhs[f], rs[f] = norm * bc[f], norm_scale * abs(bc[f])
            elif codes[f] == 2:    # PB_BC_NEU: rhs += s bc area
                rhs[f] += sign[f] * bc[f] * areas[f]
                rs[f] += abs(bc[f] * areas[f])
        self.H, self.Hs, self.rhs, self.rs = H, Hs, rhs, rs

    def recover(self, lam):
        T = self.T
        u, us = np.zeros(T.nf), np.zeros(T.nf)
        p, ps = np.zeros(T.nc), np.zeros(T.nc)
        with mp.workdps(DPS):
            for c, (E, z, t, h, Ef, kappa) in enumerate(self.cells):
                f, s = T.faces(c), T.signs(c)
                n = f.size
                lv = [mp.mpf(float(lam[x])) for x in f]
                pc = (-sum(z[j] * lv[j] for j in range(n)) - h) / t
                p[c] = float(pc)
                la, rho, Sf = np.abs(lam[f]), np.abs(Ef).sum(axis=1), abs(1 / float(t))
                zl = abs(float(sum(z[j] * lv[j] for j in range(n))))
                ps[c] = kappa * Sf * (float(rho @ la) + Sf * rho.sum() * (zl + abs(float(h))))
                for i in range(n):
                    if T.first[f[i]] != c:
                        continue
                    u[f[i]] = s[i] * float(sum(E[i, j] * (pc - lv[j]) for j in range(n)))
                    us[f[i]] = kappa * float(np.abs(Ef[i]) @ (la + abs(p[c]))) + float(np.abs(Ef[i]).sum()) * ps[c]
        return np.concatenate((u, p)), np.concatenate((us, ps))


def worst(got, ref, scale):
    """Largest |got - ref| / scale over the entries (entries of scale 0 must match exactly) and where it is."""
    got, ref, scale = (np.asarray(a, float) for a in (got, ref, scale))
    diff = np.abs(got - ref)
    assert not np.any(diff[scale == 0] != 0), "a value outside the cells' pattern"
    ratio = np.where(scale > 0, diff / np.where(scale > 0, scale, 1.0), 0.0)
    k = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    return float(ratio[k]), k
