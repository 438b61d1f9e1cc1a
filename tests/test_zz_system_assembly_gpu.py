"""The device-side flow and mechanics systems on every path they dispatch to, against extended-precision references.

``Mpfa.assemble_matrix_rhs`` / ``Mpsa.assemble_matrix_rhs`` form A = div @ flux (``div_flux_kernel``, atomics) and
A = div_nd @ stress (``div_stress_gather_kernel``, one writer per row) and their right-hand sides
(``face_row_dot_kernel`` / ``bound_stress_dot_kernel`` + ``neg_div_kernel`` / ``neg_div_nd_kernel``) in csrc/api.cu.

Every entry of A and b is checked against a sum of all its product terms accumulated in ``np.longdouble`` with the
a-priori bound ``(k + 2) u sum |terms|`` of a k-term float64 sum (the helpers of test_zz_sparse_paths_gpu.py).  The
pattern of A is checked against one built independently from the cell-node incidence ("cells sharing a node",
block-expanded), and every stored entry that no face contributes to must be exactly 0.

Sizes that must cross a branch are derived from the SM count and the launch formulas of api.cu: one warp per row
with 16 SMs CTAs of 8 warps (128 SMs rows per pass), the gather 24 SMs CTAs of 4 warps (96 SMs cells per pass), the
rhs scatters 16 SMs CTAs of 256 threads (4096 SMs faces or face components per pass), and the gather stages a row
in shared memory only up to 128 block columns.  The reference self-checks at the top run without a GPU."""
import math

import numpy as np
import pytest
import scipy.sparse as sps

import porepy_b200 as pb
from porepy_b200.grid import Grid
from test_zz_sparse_paths_gpu import LD, U, _EXTENDED, _assert_within, _exact_products, _row_sums, _spgemm_ref

K_CAP = 128          # div_stress_gather_kernel: block columns staged in shared memory per row
PATTERN_CAP = 256    # pattern_kernel: candidates per row on the device (host fallback above)


# ---------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------
def _div(sd, nd):
    """div_nd, canonical CSR: row c nd + i, column f nd + i, value cell_faces[f, c]."""
    d = sps.kron(sps.csr_matrix(sps.csc_matrix(sd.cell_faces).T), sps.identity(nd)).tocsr()
    d.sort_indices()
    return d


def _system_ref(sd, nd, m):
    """(indptr, indices, value, bound) of div_nd @ m over its structural pattern (exact cancellations kept)."""
    m = sps.csr_matrix(m)
    m.sort_indices()
    return _spgemm_ref(_div(sd, nd), m)


def _mv_terms(m, x):
    """(row, term) of every product m[r, j] x[j] of m @ x."""
    m = sps.csr_matrix(m)
    return np.repeat(np.arange(m.shape[0]), np.diff(m.indptr)), _exact_products(m.data, x[m.indices])


def _rhs_ref(sd, nd, parts, source=None):
    """(value, bound) of b = -div_nd @ (sum of the row terms in ``parts``) + source: every term of every face row,
    signed for each cell of the face, and the source, summed per row in long double."""
    dv = sps.csc_matrix(_div(sd, nd))
    rows, terms = [], []
    for mrow, t in parts:
        cnt = np.diff(dv.indptr)[mrow]
        pos = np.repeat(dv.indptr[mrow], cnt) + np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        rows.append(dv.indices[pos])
        terms.append(-dv.data[pos] * np.repeat(t, cnt))
    n = sd.num_cells * nd
    if source is not None:
        rows.append(np.arange(n)), terms.append(np.asarray(source, terms[0].dtype if terms else float))
    rows = np.concatenate(rows)
    terms = np.concatenate(terms)
    order = np.argsort(rows, kind="stable")
    indptr = np.r_[0, np.cumsum(np.bincount(rows, minlength=n))]
    val = _row_sums(terms[order], indptr)
    absum = _row_sums(np.abs(terms[order]), indptr).astype(np.float64)
    return val, (np.diff(indptr) + 2) * U * absum


def _node_pattern(sd, nd):
    """Block-expanded "cells sharing a node" from the cell-node incidence: the pattern A must have."""
    cn = (abs(sps.csr_matrix(sps.csc_matrix(sd.cell_faces).T)) @ abs(sps.csr_matrix(sps.csc_matrix(sd.face_nodes).T)))
    cn.data[:] = 1.0
    cc = (cn @ cn.T).tocsr()
    p = sps.kron(cc, np.ones((nd, nd))).tocsr()
    p.sort_indices()
    return p.indptr, p.indices


def _candidates(sd):
    """Largest candidate count of a row of the four structural patterns (sum over the row entity's nodes of the
    node's column entities), as pattern_kernel gathers them."""
    fn = abs(sps.csr_matrix(sps.csc_matrix(sd.face_nodes)))          # node x face
    cf = abs(sps.csr_matrix(sps.csc_matrix(sd.cell_faces)))          # face x cell
    cn = (cf.T @ fn.T).tocsr()
    cn.data[:] = 1.0                                                 # cell x node
    cells_of_node = np.asarray(cn.sum(axis=0)).ravel()
    bnd = np.zeros(sd.num_faces)
    bnd[sd.get_all_boundary_faces()] = 1.0
    bfaces_of_node = fn @ bnd
    fnb = fn.T.tocsr()
    fnb.data[:] = 1.0
    return int(max((x @ y).max() for x in (fnb, cn) for y in (cells_of_node, bfaces_of_node)))


# ---------------------------------------------------------------------------------------------------------------------
# triangle grids (compute_geometry is 3-D only)
# ---------------------------------------------------------------------------------------------------------------------
def _tri_geometry(g):
    """Geometry of a triangle grid in the plane z = 0: edge midpoints and lengths, normals (edge rotated by -90
    degrees) pointing out of the cell whose ``cell_faces`` entry is +1, vertex-mean cell centres, areas.  The two
    nodes of a flipped face are swapped so that the node order stays consistent with the normal."""
    fn = sps.csc_matrix(g.face_nodes)
    e = fn.indices.reshape(-1, 2)
    p = g.nodes
    a, b = p[:, e[:, 0]], p[:, e[:, 1]]
    t = b - a
    nrm = np.vstack([t[1], -t[0], np.zeros(t.shape[1])])
    fc = 0.5 * (a + b)
    fa = np.linalg.norm(t, axis=0)
    cf = sps.csc_matrix(g.cell_faces)
    cnodes = (abs(cf.T) @ abs(fn.T)).tocsr()
    cnodes.sort_indices()
    tri = cnodes.indices.reshape(-1, 3)
    cc = p[:, tri].mean(axis=2)
    u, v = p[:, tri[:, 1]] - p[:, tri[:, 0]], p[:, tri[:, 2]] - p[:, tri[:, 0]]
    cv = 0.5 * np.abs(u[0] * v[1] - u[1] * v[0])
    coo = sps.coo_matrix(cf)
    cell = coo.col[np.argsort(coo.row, kind="stable")]
    sgn = coo.data[np.argsort(coo.row, kind="stable")]
    first = np.r_[0, np.cumsum(np.bincount(coo.row, minlength=g.num_faces))[:-1]]
    ref_cell, ref_sgn = cell[first], sgn[first]
    outward = np.einsum("ij,ij->j", nrm, fc - cc[:, ref_cell]) * ref_sgn
    flip = outward < 0
    nrm[:, flip] *= -1.0
    fn.indices.reshape(-1, 2)[flip] = e[flip][:, ::-1]
    g.face_nodes = fn
    return g.set_geometry(nrm, fc, fa, cc, cv)


def _tri_grid(xy, tris):
    """A conforming triangle grid from node coordinates (2, nn) and a cell-node table (nc, 3)."""
    nn, nc = xy.shape[1], tris.shape[0]
    nodes = np.vstack([xy, np.zeros(nn)])
    edges = np.sort(tris[:, [[0, 1], [1, 2], [2, 0]]].reshape(-1, 2), axis=1)
    uniq, inv = np.unique(edges[:, 0].astype(np.int64) * nn + edges[:, 1], return_inverse=True)
    nf = uniq.size
    fnodes = np.stack([uniq // nn, uniq % nn], axis=1)
    face_nodes = sps.csc_matrix((np.ones(2 * nf, bool), fnodes.ravel(), np.arange(0, 2 * nf + 1, 2)), shape=(nn, nf))
    # sign: +1 where the rotated edge (b - a) points out of the cell
    a, b = nodes[:, fnodes[inv, 0]], nodes[:, fnodes[inv, 1]]
    cc = np.repeat(nodes[:, tris].mean(axis=2), 3, axis=1)
    out = (b[1] - a[1]) * (0.5 * (a[0] + b[0]) - cc[0]) - (b[0] - a[0]) * (0.5 * (a[1] + b[1]) - cc[1])
    cell_faces = sps.csc_matrix((np.where(out > 0, 1.0, -1.0), inv, np.arange(0, 3 * nc + 1, 3)), shape=(nf, nc))
    cell_faces.sort_indices()
    return _tri_geometry(Grid(2, nodes, face_nodes, cell_faces, name="TriangleGrid"))


def _fan_grid(m):
    """A centre node with m triangles around it (rim radius 1) and a ring of 2 m triangles outside: the centre
    node's m cells share it, so each of their CELL x CELL rows holds m + 5 cells."""
    th = 2 * np.pi * np.arange(m) / m
    r_out = 1.0 + 2 * np.pi / m
    xy = np.hstack([[[0.0], [0.0]], np.vstack([np.cos(th), np.sin(th)]),
                    r_out * np.vstack([np.cos(th + np.pi / m), np.sin(th + np.pi / m)])])
    i = np.arange(m)
    rim, nxt, out, onx = 1 + i, 1 + (i + 1) % m, 1 + m + i, 1 + m + (i + 1) % m
    tris = np.vstack([np.stack([np.zeros(m, int), rim, nxt], 1), np.stack([rim, nxt, out], 1),
                      np.stack([nxt, onx, out], 1)])
    return _tri_grid(xy, tris)


def _square_tri_grid(nx, ny, seed=0):
    """nx x ny squares of the unit square, each cut into two triangles, interior nodes perturbed."""
    rng = np.random.default_rng(seed)
    x, y = np.meshgrid(np.linspace(0, 1, nx + 1), np.linspace(0, 1, ny + 1), indexing="ij")
    x, y = x.ravel(order="F"), y.ravel(order="F")
    inner = (x > 0) & (x < 1) & (y > 0) & (y < 1)
    x[inner] += 0.25 / nx * (rng.random(inner.sum()) - 0.5)
    y[inner] += 0.25 / ny * (rng.random(inner.sum()) - 0.5)
    i, j = (a.ravel(order="F") for a in np.meshgrid(np.arange(nx), np.arange(ny), indexing="ij"))
    n0 = i + (nx + 1) * j
    n1, n2, n3 = n0 + 1, n0 + nx + 2, n0 + nx + 1
    tris = np.vstack([np.stack([n0, n1, n2], 1), np.stack([n0, n2, n3], 1)])
    return _tri_grid(np.vstack([x, y]), tris)


def _tilted(g, seed=0):
    """The 2-D grid g rotated into a tilted plane of 3-D (a fracture plane); areas and volumes are unchanged."""
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
    t = Grid(2, q @ g.nodes, g.face_nodes, g.cell_faces, name=g.name)
    return t.set_geometry(q @ g.face_normals, q @ g.face_centers, g.face_areas, q @ g.cell_centers, g.cell_volumes)


# ---------------------------------------------------------------------------------------------------------------------
# 1. self-checks of the references (no GPU)
# ---------------------------------------------------------------------------------------------------------------------
def _emu_plan(g):
    import emu_binding
    return emu_binding.EmuPlan(g)


def _emu_mpsa(g, seed=0):
    rng = np.random.default_rng(seed)
    nd, nc, nf = g.dim, g.num_cells, g.num_faces
    c = pb.FourthOrderTensor(np.exp(0.4 * rng.standard_normal(nc)), np.exp(0.4 * rng.standard_normal(nc)))
    codes = np.zeros((nd, nf), np.uint8)
    bf = g.get_all_boundary_faces()
    codes[:, bf] = np.where(np.arange(bf.size) % 3 == 0, 1, 2)
    from porepy_b200 import fv
    return _emu_plan(g).mpsa(c.values, codes, None, fv.determine_eta(g))


def _emu_mpfa(g, seed=0):
    rng = np.random.default_rng(seed)
    nc, nf = g.num_cells, g.num_faces
    k = pb.SecondOrderTensor(1 + rng.random(nc), 1 + rng.random(nc), 1 + rng.random(nc), 0.3 * rng.random(nc),
                             0.3 * rng.random(nc) * (g.dim == 3), 0.3 * rng.random(nc) * (g.dim == 3))
    codes = np.zeros(nf, np.uint8)
    bf = g.get_all_boundary_faces()
    codes[bf] = np.where(np.arange(bf.size) % 3 == 0, 1, 2)
    from porepy_b200 import fv
    return _emu_plan(g).mpfa(k.values, codes, None, fv.determine_eta(g))


def test_system_reference_against_fsum():
    """The long-double div_nd @ stress and -div_nd @ (bound_stress @ bc) + source of a small grid equal the
    correctly rounded sums (math.fsum of the exact terms) within one rounding."""
    g = pb.cart_grid_3d([3, 3, 2], perturb=0.3, seed=1)
    out = _emu_mpsa(g)
    m = out["stress"].tocsr()
    ip, ix, vals, bound = _system_ref(g, 3, m)
    div = _div(g, 3).toarray()
    dense = m.toarray()
    rows = np.repeat(np.arange(ip.size - 1), np.diff(ip))
    for q in range(0, ix.size, 7):
        terms = div[rows[q]] * dense[:, ix[q]]
        exact = math.fsum(terms)
        assert abs(float(vals[q] - LD(exact))) <= 1.01 * U * abs(exact) + 1e-300
        assert bound[q] >= U * np.abs(terms).sum()
    assert vals.size == np.count_nonzero((abs(sps.csr_matrix(div)) @ abs(sps.csr_matrix(dense).astype(bool)
                                                                        .astype(float))).toarray())
    rng = np.random.default_rng(2)
    bc, src = rng.standard_normal(3 * g.num_faces), rng.standard_normal(3 * g.num_cells)
    bs = out["bound_stress"].tocsr()
    val, bnd = _rhs_ref(g, 3, [_mv_terms(bs, bc)], src)
    bsd = bs.toarray()
    for r in range(3 * g.num_cells):
        terms = np.r_[(-div[r][:, None] * bsd * bc[None, :]).ravel(), src[r]]
        exact = math.fsum(terms)              # of the float64-rounded products: one rounding each
        assert abs(float(val[r] - LD(exact))) <= 1.01 * U * (abs(exact) + np.abs(terms).sum()) + 1e-300, r
        assert bnd[r] >= U * np.abs(terms).sum()


@pytest.mark.parametrize("make", [lambda: pb.cart_grid_3d([4, 3, 3], perturb=0.3, seed=2),
                                  lambda: pb.structured_tet_grid([2, 2, 2]),
                                  lambda: _square_tri_grid(5, 4), lambda: _fan_grid(20), lambda: pb.cart_grid_2d([5, 4])],
                         ids=["cart3d", "tet3d", "tri2d", "fan20", "cart2d"])
def test_node_pattern_contains_every_structural_entry(make):
    """The host build's MPSA stress and MPFA flux: every structural entry of div_nd @ M lies in the "cells sharing a
    node" pattern, and the diagonal blocks are full."""
    g = make()
    nd = g.dim
    for m, bs in ((_emu_mpsa(g)["stress"], nd), (_emu_mpfa(g)["flux"], 1)):
        ip, ix, _, _ = _system_ref(g, bs, m)
        pip, pix = _node_pattern(g, bs)
        n = pip.size - 1
        key = np.repeat(np.arange(n), np.diff(ip)) * n + ix
        pkey = np.repeat(np.arange(n), np.diff(pip)) * n + pix
        assert np.isin(key, pkey).all()
        diag = np.repeat(np.arange(n), bs) * n + (np.arange(n)[:, None] // bs * bs + np.arange(bs)).ravel()
        assert np.isin(diag, key).all()


def test_triangle_geometry_matches_the_golden():
    """_tri_geometry on the topology of the mpfa_tri2d fixture reproduces the reference geometry."""
    from golden_io import load_case
    c = load_case("mpfa_tri2d")
    ref = c.g
    g = Grid(2, ref.nodes, sps.csc_matrix(ref.face_nodes, copy=True), ref.cell_faces, name=ref.name)
    _tri_geometry(g)
    for key in ("face_normals", "face_centers", "face_areas", "cell_centers", "cell_volumes"):
        assert np.abs(getattr(g, key) - getattr(ref, key)).max() <= 1e-14, key


@pytest.mark.parametrize("m", [140, 300])
def test_fan_grid(m):
    g = _fan_grid(m)
    assert (g.num_cells, g.num_nodes, g.num_faces) == (3 * m, 2 * m + 1, 5 * m)
    assert g.cell_volumes.min() > 0 and abs(g.cell_volumes.sum() - np.pi * (1 + 2 * np.pi / m) ** 2) < 0.05
    assert g.get_all_boundary_faces().size == m
    # the signed normals of each cell sum to zero (a closed cell) and point out of the cell with sign +1
    cf = sps.coo_matrix(g.cell_faces)
    assert np.abs(g.face_normals @ sps.csc_matrix(g.cell_faces)).max() < 1e-12
    dots = np.einsum("ij,ij->j", g.face_normals[:, cf.row], g.face_centers[:, cf.row] - g.cell_centers[:, cf.col])
    assert np.all(dots * cf.data > 0)
    ip, _ = _node_pattern(g, 1)
    assert np.diff(ip)[:m].min() == m + 5 and np.diff(ip).max() == m + 5
    assert (_candidates(g) <= PATTERN_CAP) == (m == 140)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the checks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _check_matrix(sd, nd, a_dev, m, what):
    """A (a DeviceCsr) has exactly the node pattern; on the structural entries of div_nd @ m it is within the bound
    of the long-double sum; every other stored entry is exactly 0."""
    a = a_dev.to_scipy()
    n = sd.num_cells * nd
    assert a.shape == (n, n), what
    pip, pix = _node_pattern(sd, nd)
    assert np.array_equal(a.indptr, pip) and np.array_equal(a.indices, pix), f"{what}: pattern"
    ip, ix, vals, bound = _system_ref(sd, nd, m)
    key = np.repeat(np.arange(n, dtype=np.int64), np.diff(ip)) * n + ix
    akey = np.repeat(np.arange(n, dtype=np.int64), np.diff(a.indptr)) * n + a.indices
    pos = np.searchsorted(akey, key)
    assert np.array_equal(akey[np.minimum(pos, akey.size - 1)], key), f"{what}: a structural entry is not stored"
    _assert_within(a.data[pos], vals, bound, what)
    rest = np.ones(akey.size, bool)
    rest[pos] = False
    assert not a.data[rest].any(), f"{what}: {np.count_nonzero(a.data[rest])} entries without a face term are not 0"
    return a


def _assert_bitwise(a, b, what):
    assert np.array_equal(a.data.view(np.int64), b.to_scipy().data.view(np.int64)), f"{what}: not bit-identical"


def _vector_bc(g, rng):
    """Dirichlet on x = 0, Robin (anisotropic weight) on x = 1, a roller in a rotated basis on y = 0, Neumann
    elsewhere; a rotated basis on the Dirichlet faces too."""
    nd, nf = g.dim, g.num_faces
    bf = g.get_all_boundary_faces()
    x, y = g.face_centers[0, bf], g.face_centers[1, bf]
    bc = pb.BoundaryConditionVectorial(g)
    for faces, kind in ((bf[x < 1e-10], "dir"), (bf[x > 1 - 1e-10], "rob")):
        bc.is_neu[:, faces] = False
        getattr(bc, "is_" + kind)[:, faces] = True
    roll = bf[(y < 1e-10) & (x > 1e-10) & (x < 1 - 1e-10)]
    bc.is_neu[0, roll] = False
    bc.is_dir[0, roll] = True
    w = rng.uniform(0.5, 2.0, (nd, nd, nf))
    bc.robin_weight = 0.5 * (w + w.transpose(1, 0, 2)) + 2 * np.eye(nd)[:, :, None]
    for faces in (roll, bf[x < 1e-10][::2]):
        for f in faces:
            q, _ = np.linalg.qr(rng.standard_normal((nd, nd)))
            bc.basis[:, :, f] = q
    return bc


def _scalar_bc(g, rng):
    bf = g.get_all_boundary_faces()
    x = g.face_centers[0, bf]
    lab = np.where(x < 1e-10, "dir", np.where(x > 1 - 1e-10, "rob", "neu"))
    bc = pb.BoundaryCondition(g, bf, list(lab))
    bc.robin_weight = rng.uniform(0.5, 2.0, g.num_faces)
    return bc


def _aniso(g, rng):
    nc = g.num_cells
    off = 0.3 * rng.random((3, nc))
    if g.dim == 2:
        off[1:] = 0.0
    return pb.SecondOrderTensor(1 + rng.random(nc), 1 + rng.random(nc), 1 + rng.random(nc), *off)


def _stiffness(g, rng):
    nc = g.num_cells
    return pb.FourthOrderTensor(np.exp(0.5 * rng.standard_normal(nc)), np.exp(0.5 * rng.standard_normal(nc)))


def _mechanics(g, rng, keyword="mech", cls=pb.Mpsa, **extra):
    """Discretize, then assemble on the device while the matrices are device resident; returns the device system,
    the rhs (with source), the rhs without source, a repeat of the system, and the downloaded matrices."""
    nd, nc, nf = g.dim, g.num_cells, g.num_faces
    bv, src = rng.standard_normal(nd * nf), rng.standard_normal(nd * nc)
    data = pb.initialize_data({}, keyword, {"fourth_order_tensor": _stiffness(g, rng), "bc": _vector_bc(g, rng),
                                            "bc_values": bv, "source": src, **extra})
    d = cls(keyword)
    d.discretize(g, data)
    mats = data[pb.DISCRETIZATION_MATRICES][keyword]
    stress, bstress = mats["stress"], mats["bound_stress"]
    plan = stress.plan
    if cls is pb.Mpsa:
        a_dev, b = d.assemble_matrix_rhs_device(g, data)
    else:                       # Biot assembles through the plan
        a_dev = plan.mpsa_system(stress.device_values)
        b = plan.mpsa_rhs(bv, src, bound_stress=bstress.device_values)
    again = plan.mpsa_system(stress.device_values)
    b0 = plan.mpsa_rhs(bv, None, bound_stress=bstress.device_values)
    return dict(a=a_dev, b=b, b0=b0, again=again, handle=stress.device_values, stress=sps.csr_matrix(stress),
                bstress=sps.csr_matrix(bstress), bv=bv, src=src, plan=plan)


def _check_mechanics(g, r, what):
    nd = g.dim
    a = _check_matrix(g, nd, r["a"], r["stress"], what)
    _assert_bitwise(a, r["again"], what)
    terms = [_mv_terms(r["bstress"], r["bv"])]
    for b, src, tag in ((r["b"], r["src"], "b"), (r["b0"], None, "b without source")):
        val, bound = _rhs_ref(g, nd, terms, src)
        _assert_within(b, val, bound, f"{what} {tag}")
    return a


def _flow(g, rng, amb=None):
    """MPFA with bc values and a vector source; the device system and rhs, the rhs without the vector source and
    the downloaded matrices."""
    nc, nf = g.num_cells, g.num_faces
    amb = amb or g.dim
    bv, vs = rng.standard_normal(nf), rng.standard_normal(amb * nc)
    prm = {"second_order_tensor": _aniso(g, rng), "bc": _scalar_bc(g, rng), "bc_values": bv, "vector_source": vs}
    if amb != g.dim:
        prm["ambient_dimension"] = amb
    data = pb.initialize_data({}, "flow", prm)
    d = pb.Mpfa("flow")
    d.discretize(g, data)
    mats = data[pb.DISCRETIZATION_MATRICES]["flow"]
    a_dev, b = d.assemble_matrix_rhs_device(g, data)
    plan = mats["flux"].plan
    b0 = plan.mpfa_rhs(bv, None, bound_flux=mats["bound_flux"].device_values)
    vsd = mats["vector_source"]
    inplane = vsd.device_values.download() if g.dim == 2 and amb == 3 or plan.rotation is not None else None
    return dict(a=a_dev, b=b, b0=b0, flux=sps.csr_matrix(mats["flux"]), bflux=sps.csr_matrix(mats["bound_flux"]),
                vsd=sps.csr_matrix(vsd), inplane=inplane, bv=bv, vs=vs, amb=amb, plan=plan)


def _check_flow(g, r, what):
    a = _check_matrix(g, 1, r["a"], r["flux"], what)
    bterms = _mv_terms(r["bflux"], r["bv"])
    val, bound = _rhs_ref(g, 1, [bterms])
    _assert_within(r["b0"], val, bound, f"{what} b without vector source")
    if r["inplane"] is None:
        vterms = _mv_terms(r["vsd"], r["vs"])
    else:
        # the device holds the in-plane coefficients d_a and gets the vector rotated into the plane: the terms are
        # d_a R_ab v_b over the two in-plane components a and the ambient components b
        amb, plan = r["amb"], r["plan"]
        rows = (np.eye(3) if plan.rotation is None else plan.rotation)[:2, :amb]
        ip, ix = plan.base_pattern(0)
        d = r["inplane"].reshape(-1, 2)
        face = np.repeat(np.arange(ip.size - 1), np.diff(ip))
        v = np.asarray(r["vs"], LD).reshape(-1, amb)[ix]                              # (nnz, amb)
        t = np.asarray(d, LD)[:, :, None] * np.asarray(rows, LD)[None] * v[:, None, :]  # (nnz, 2, amb)
        vterms = (np.repeat(face, 2 * amb), t.ravel() if _EXTENDED else t.astype(np.float64).ravel())
        # and the host's lifted (ambient) matrix gives the same product
        host = -_div(g, 1) @ (r["vsd"] @ r["vs"])
        ref_v, _ = _rhs_ref(g, 1, [vterms])
        assert np.abs(host - ref_v.astype(np.float64)).max() <= 1e-12 * max(np.abs(host).max(), 1.0)
    val, bound = _rhs_ref(g, 1, [bterms, vterms])
    _assert_within(r["b"], val, bound, f"{what} b")
    return a


# ---------------------------------------------------------------------------------------------------------------------
# 2. 3-D, with the grid-stride wraps of the one-warp-per-row kernels and of the gather
# ---------------------------------------------------------------------------------------------------------------------
_GRIDS = {}


def _grid3d(name, sm):
    if name not in _GRIDS:
        if name == "cart-wrap":          # more cells than one pass of 128 SMs warps
            n = int(math.ceil((128 * sm) ** (1 / 3))) + 1
            _GRIDS[name] = pb.cart_grid_3d([n, n - 1, n - 1], perturb=0.3, seed=4)
        else:
            _GRIDS[name] = pb.structured_tet_grid([9, 8, 7])
    return _GRIDS[name]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cart-wrap", "tet"])
def test_mechanics_system_3d(name, sm):
    g = _grid3d(name, sm)
    if name == "cart-wrap":
        assert g.num_cells > 128 * sm and g.num_cells > 96 * sm and 3 * g.num_faces > 128 * sm
    r = _mechanics(g, np.random.default_rng(30))
    assert np.diff(r["plan"].base_pattern(2)[0]).max() <= K_CAP
    print(f"mechanics {name}: {g.num_cells} cells, nnz {r['a'].nnz}")
    _check_mechanics(g, r, f"mechanics {name}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cart-wrap", "tet"])
def test_flow_system_3d(name, sm):
    g = _grid3d(name, sm)
    if name == "cart-wrap":
        assert g.num_faces > 128 * sm
    r = _flow(g, np.random.default_rng(31))
    _check_flow(g, r, f"flow {name}")


# ---------------------------------------------------------------------------------------------------------------------
# 3. the rhs scatters past one pass of their grids (2-D)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rhs_scatter_wraps(sm):
    n = int(math.sqrt(2048 * sm)) + 4
    g = pb.cart_grid_2d([n, n])
    assert g.num_faces > 4096 * sm and 2 * g.num_faces > 4096 * sm
    rng = np.random.default_rng(32)
    nc, nf = g.num_cells, g.num_faces
    bv, src = rng.standard_normal(2 * nf), rng.standard_normal(2 * nc)
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": _stiffness(g, rng), "bc": _vector_bc(g, rng),
                                           "bc_values": bv, "source": src})
    pb.Mpsa("mech").discretize(g, data)
    mats = data[pb.DISCRETIZATION_MATRICES]["mech"]
    b = mats["stress"].plan.mpsa_rhs(bv, src, bound_stress=mats["bound_stress"].device_values)
    val, bound = _rhs_ref(g, 2, [_mv_terms(sps.csr_matrix(mats["bound_stress"]), bv)], src)
    _assert_within(b, val, bound, "mechanics rhs")
    fbv = rng.standard_normal(nf)
    data = pb.initialize_data({}, "flow", {"second_order_tensor": _aniso(g, rng), "bc": _scalar_bc(g, rng),
                                           "bc_values": fbv})
    pb.Mpfa("flow").discretize(g, data)
    mats = data[pb.DISCRETIZATION_MATRICES]["flow"]
    b = mats["flux"].plan.mpfa_rhs(fbv, None, bound_flux=mats["bound_flux"].device_values)
    val, bound = _rhs_ref(g, 1, [_mv_terms(sps.csr_matrix(mats["bound_flux"]), fbv)])
    _assert_within(b, val, bound, "flow rhs")


# ---------------------------------------------------------------------------------------------------------------------
# 4. 2-D: nd = 2 mechanics, flow, and the vector source rotated into the plane
# ---------------------------------------------------------------------------------------------------------------------
_MAKE_2D = {"cart2d": lambda: pb.cart_grid_2d([23, 17]), "tri2d": lambda: _square_tri_grid(14, 11, seed=3)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_MAKE_2D))
def test_mechanics_system_2d(name):
    g = _MAKE_2D[name]()
    _check_mechanics(g, _mechanics(g, np.random.default_rng(40)), f"mechanics {name}")


@pytest.mark.gpu
@pytest.mark.parametrize("amb", [2, 3])
@pytest.mark.parametrize("name", list(_MAKE_2D))
def test_flow_system_2d(name, amb):
    g = _MAKE_2D[name]()
    r = _flow(g, np.random.default_rng(41), amb=amb)
    assert (r["inplane"] is not None) == (amb == 3)
    _check_flow(g, r, f"flow {name} ambient {amb}")


@pytest.mark.gpu
@pytest.mark.parametrize("amb", [2, 3])
def test_flow_system_on_a_tilted_plane(amb):
    g = _tilted(_square_tri_grid(12, 9, seed=5), seed=6)
    r = _flow(g, np.random.default_rng(42), amb=amb)
    assert r["plan"].rotation is not None and r["inplane"] is not None
    _check_flow(g, r, f"flow tilted ambient {amb}")


# ---------------------------------------------------------------------------------------------------------------------
# 5. rows longer than the shared-memory stage of the gather (fans of 140 and 300 triangles)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("m", [140, 300])
def test_systems_with_rows_beyond_the_gather_stage(m):
    g = _fan_grid(m)
    assert (_candidates(g) <= PATTERN_CAP) == (m == 140)    # device patterns at 140, host fallback at 300
    rng = np.random.default_rng(50 + m)
    r = _mechanics(g, rng)
    lens = np.diff(r["plan"].base_pattern(2)[0])
    assert lens.max() > K_CAP and lens.min() <= K_CAP        # both branches of the gather in one launch
    _check_mechanics(g, r, f"mechanics fan {m}")
    nc = g.num_cells
    alpha = pb.SecondOrderTensor(0.5 + rng.random(nc), 0.5 + rng.random(nc), np.ones(nc), 0.2 * rng.random(nc))
    rb = _mechanics(g, rng, keyword="biot", cls=pb.Biot, scalar_vector_mappings={"p": alpha})
    _check_mechanics(g, rb, f"Biot stress fan {m}")
    _check_flow(g, _flow(g, rng), f"flow fan {m}")


# ---------------------------------------------------------------------------------------------------------------------
# 6. value handles: an explicit handle vs. the plan's last assembled array
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_mechanics_system_follows_the_given_values():
    """Keyword 1 is discretized through ``Mpsa`` (its values leave the plan as a handle), then keyword 2 is assembled
    on the same plan: ``mpsa_system(handle of 1)`` gives the system of 1, ``mpsa_system()`` that of 2."""
    from porepy_b200 import fv
    g = pb.cart_grid_3d([6, 5, 4], perturb=0.3, seed=7)
    rng = np.random.default_rng(60)
    r1 = _mechanics(g, rng, keyword="one")
    plan = r1["plan"]
    assert pb.DevicePlan.for_grid(g) is plan
    c2, bc2 = _stiffness(g, rng), _vector_bc(g, rng)
    codes, robw = fv.vector_bc_codes(bc2, 3, g.num_faces)
    plan.mpsa_upload(c2.values, codes, robw, 0.0)
    plan.mpsa_set_basis(fv.vector_bc_basis(bc2, 3, codes))
    plan.mpsa_assemble()
    a_last = plan.mpsa_system()
    a_first = plan.mpsa_system(r1["handle"])
    bv = rng.standard_normal(3 * g.num_faces)
    b_last = plan.mpsa_rhs(bv)
    m2 = plan.mpsa_download()
    _check_matrix(g, 3, a_first, r1["stress"], "explicit handle")
    _check_matrix(g, 3, a_last, m2["stress"], "last assembled")
    val, bound = _rhs_ref(g, 3, [_mv_terms(m2["bound_stress"], bv)])
    _assert_within(b_last, val, bound, "rhs of the last assembled")


# ---------------------------------------------------------------------------------------------------------------------
# 7. a sharded mechanics system, two shards one after the other on one GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_sharded_mechanics_system():
    """Each shard assembles only its own nodes (``set_active_nodes``); shard 0 gets the stiffness restricted on the
    host, shard 1 the global tensor through the cell map.  Each shard's A and b match the long-double reference of
    its own matrices, and its own-cell rows match the unsplit system."""
    from porepy_b200 import shard as sh
    g = pb.cart_grid_3d([8, 7, 6], perturb=0.3, seed=8)
    rng = np.random.default_rng(70)
    nd, nc, nf = 3, g.num_cells, g.num_faces
    c, vbc = _stiffness(g, rng), _vector_bc(g, rng)
    bv, src = rng.standard_normal(nd * nf), rng.standard_normal(nd * nc)
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": c, "bc": vbc, "bc_values": bv, "source": src})
    d = pb.Mpsa("mech")
    d.discretize(g, data)
    a_full, b_full = d.assemble_matrix_rhs_device(g, data)
    a_full = a_full.to_scipy()
    part = sh.partition_cells(g, 2)
    blk = lambda cells: (cells[:, None] * nd + np.arange(nd)).ravel()  # noqa: E731
    for rank in range(2):
        s = sh.extract_shard(g, part, rank)
        n_own = int(s.own_cell.sum())
        assert s.own_cell[:n_own].all() and not s.own_cell[n_own:].any()
        plan = pb.DevicePlan.for_grid(s.grid)
        plan.set_active_nodes(s.own_node)
        if rank == 1:
            plan.set_cell_map(s.cells, nc)
        cl = c if rank == 1 else pb.FourthOrderTensor.from_values(s.restrict_cell_array(c.values))
        bl, sl = bv.reshape(nf, nd)[s.faces].ravel(), src.reshape(nc, nd)[s.cells].ravel()
        dl = pb.initialize_data({}, "mech", {"fourth_order_tensor": cl, "bc": sh.restrict_vector_bc(vbc, s),
                                             "bc_values": bl, "source": sl, "mpsa_eta": pb.determine_eta(g)})
        dd = pb.Mpsa("mech")
        dd.discretize(s.grid, dl)
        a_dev, b_loc = dd.assemble_matrix_rhs_device(s.grid, dl)
        mats = dl[pb.DISCRETIZATION_MATRICES]["mech"]
        stress, bstress = sps.csr_matrix(mats["stress"]), sps.csr_matrix(mats["bound_stress"])
        _check_matrix(s.grid, nd, a_dev, stress, f"shard {rank}")
        val, bound = _rhs_ref(s.grid, nd, [_mv_terms(bstress, bl)], sl)
        _assert_within(b_loc, val, bound, f"shard {rank} b")
        rows = a_dev.truncate_rows(n_own * nd).to_scipy()
        ref = a_full[blk(s.cells[:n_own])][:, blk(s.cells)]
        assert abs(ref - rows).max() <= 1e-12 * abs(a_full).max(), rank
        assert np.abs(b_loc[:n_own * nd] - b_full[blk(s.cells[:n_own])]).max() <= 1e-12 * np.abs(b_full).max(), rank
