"""The mixed schemes and the 3-D geometry on polygonal and polyhedral cells, entry by entry against an
extended-precision restatement (tests/dual_mp.py).

``dual_kernel`` (csrc/dual.cu) runs MVEM on cells with any number of faces, ``hybrid_cell_kernel`` condenses cells of
up to 32 faces with one warp lane per face, and ``geom_face`` / ``geom_cell`` fan faces and cells of any size.  Here:

- every ``dual_*`` and ``hybrid_*`` fixture (the agglomerated polygons and polyhedra of tools/make_dual_golden.py among
  them) on the host build and on the device, each value against mpmath at 40 digits with its own error scale, so that
  the cells of permeability 10^6 are held to the same relative accuracy as those of permeability 1;
- one star-shaped polygon of every face count from 3 to 32 (MVEM and the hybridization), 40 and 64 (MVEM only), and
  on the device one grid of all of them, so that one launch mixes every cell size up to the 32-face shared-memory
  layout;
- the refusals: two 130-gons sharing an edge (more than 256 faces in one mass row) and non-convex polyhedra, whose
  fan from the temporary centre has negative sub-tetrahedra (the reference raises the same error on both shapes);
- bit-identical repeats of the condensation and the recovery on the device."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sps

import porepy_b200 as pb
from porepy_b200 import fv
from porepy_b200.grid import Grid, cart_grid_3d
import dual_mp as D
from emu_dual_hybrid import EmuHybridDualGrid
from golden_io import case_names, load_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from agglomerate import agglomerate  # noqa: E402

BACKENDS = ["host", pytest.param("gpu", marks=pytest.mark.gpu)]
SWEEP = list(range(3, 33))


def handle(backend, g):
    """The host build of the routines or the device handle, behind the same ``DualGrid`` calls."""
    return EmuHybridDualGrid(g) if backend == "host" else fv.DualGrid(g)


def dual_inputs(g, K):
    """What ``MVEM.discretize`` / ``RT0.discretize`` hand the kernel: geometry and tensor in the grid's frame."""
    rot = fv.dual_frame(g)
    geo = [rot @ np.asarray(a, float) for a in (g.nodes, g.face_normals, g.face_centers, g.cell_centers)]
    return geo + [np.asarray(g.cell_volumes, float)], fv.rotate_second_order(K, rot), rot


def check_mass(dg, g, method, K):
    geo, perm, rot = dual_inputs(g, K)
    bad, _ = dg.discretize(method, geo, perm, rot)
    assert bad == -1
    mass, proj = dg.download()
    ip, ix = dg.mass_pattern()
    M, Ms, P, Ps = D.mass_reference(g, method, geo, perm, rot)
    r, at = D.worst(sps.csr_matrix((mass, ix, ip), shape=(g.num_faces, g.num_faces)).toarray(), M, Ms)
    assert r <= D.MASS_TOL, ("mass", r, at)
    r, at = D.worst(proj, P, Ps)
    assert r <= D.PROJ_TOL, ("vector_proj", r, at)


def hybrid_inputs(g, data):
    return pb.HybridDualVEM("flow")._inputs(g, data)


def check_hybrid(dg, g, data):
    """H and its right-hand side, then p and u from the face pressures of a solve of H: the returned values."""
    geo, codes, values = hybrid_inputs(g, data)
    H, rhs, bad, _ = dg.hybrid_system(0, geo, codes, np.zeros(g.num_faces), g.face_areas, values)
    assert bad == -1
    H = H.to_scipy().toarray()
    R = D.HybridReference(g, geo, codes, values)
    r, at = D.worst(H, R.H, R.Hs)
    assert r <= D.HYBRID_TOL, ("H", r, at)
    r, at = D.worst(rhs, R.rhs, R.rs)
    assert r <= D.HYBRID_TOL, ("rhs", r, at)
    lam = np.linalg.solve(H, rhs)
    up, _ = dg.hybrid_recover(0, geo, codes, values, lam)
    U, Us = R.recover(lam)
    r, at = D.worst(up, U, Us)
    assert r <= D.HYBRID_TOL, ("u, p", r, at)
    return H, rhs, up


def hybrid_data(c):
    return pb.initialize_data({}, "flow", {
        "second_order_tensor": pb.SecondOrderTensor.from_values(c.raw["K"]), "bc": c.bc,
        "bc_values": c.raw["bc_values"], "source": c.raw["source"], "aperture": c.raw["aperture"]})


# ------------------------------------------------------------------------------------------------------------------
# the fixtures
# ------------------------------------------------------------------------------------------------------------------


def test_polytopal_fixtures_have_the_cells_they_promise():
    for name in ("dual_mvem_poly2d", "dual_mvem_poly_plane_tilted", "hybrid_poly2d"):
        g = load_case(name).g
        n = np.diff(sps.csc_matrix(g.cell_faces).indptr)
        assert {4, 6, 8, 10, 12, 16, 32} <= set(n), (name, n)
    g = load_case("dual_mvem_poly2d").g
    # the U-shaped cell (16 edges): its centroid lies in the notch, outside the cell
    c = int(np.flatnonzero(np.diff(sps.csc_matrix(g.cell_faces).indptr) == 16)[0])
    notch = np.flatnonzero(np.diff(sps.csc_matrix(g.cell_faces).indptr) == 6)
    x = g.cell_centers[:2, c]
    assert np.any(np.abs(g.cell_centers[:2, notch] - x[:, None]).max(axis=0) < 0.1)
    for name in ("dual_mvem_poly3d", "hybrid_poly3d", "geom_poly3d"):
        g = load_case(name).g
        n = np.diff(sps.csc_matrix(g.cell_faces).indptr)
        assert {6, 10, 24, 32} == set(n), (name, n)
        assert {4, 8, 10} == set(np.diff(sps.csc_matrix(g.face_nodes).indptr)), name
        assert np.all(n[:4] != n[1:5])   # the first warps of a block hold cells of different sizes


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("name", case_names("dual_"))
def test_mass_matches_extended_precision(name, backend):
    c = load_case(name)
    check_mass(handle(backend, c.g), c.g, {"mvem": 0, "rt0": 1}[c.kind], c.raw["K"])


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("name", case_names("hybrid_"))
def test_hybridization_matches_extended_precision(name, backend):
    c = load_case(name)
    check_hybrid(handle(backend, c.g), c.g, hybrid_data(c))


@pytest.mark.gpu
def test_device_hybridization_repeats_bit_for_bit():
    c = load_case("hybrid_poly3d")
    g = c.g
    geo, codes, values = hybrid_inputs(g, hybrid_data(c))
    dg = fv.DualGrid(g)
    runs = []
    for _ in range(2):
        H, rhs, _, _ = dg.hybrid_system(0, geo, codes, np.zeros(g.num_faces), g.face_areas, values)
        H = H.to_scipy()
        lam = np.linalg.solve(H.toarray(), rhs) if not runs else runs[0][3]
        up, _ = dg.hybrid_recover(0, geo, codes, values, lam)
        runs.append((H.data, H.indices, rhs, lam, up))
    for a, b in zip(*runs):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------------------------
# polygons of 3 to 64 faces
# ------------------------------------------------------------------------------------------------------------------


def polygon_grid(loops, xy):
    """2-D grid of the counter-clockwise node loops ``loops`` over the points ``xy`` (2, n), with its geometry by the
    shoelace formulas: faces are the distinct edges (normal (dy, -dx) along the edge's first traversal), face centres
    the midpoints, cell centres the polygons' centroids."""
    edges, cf_rows, cf_cols, cf_vals = {}, [], [], []
    for c, lp in enumerate(loops):
        for a, b in zip(lp, np.roll(lp, -1)):
            key = (min(a, b), max(a, b))
            if key not in edges:
                edges[key] = (len(edges), a, b)
            f, a0, _ = edges[key]
            cf_rows.append(f)
            cf_cols.append(c)
            cf_vals.append(1.0 if a0 == a else -1.0)
    nf, nc = len(edges), len(loops)
    ends = np.array([(a, b) for _, a, b in sorted(edges.values())]).T
    nodes = np.vstack((xy, np.zeros(xy.shape[1])))
    fn = sps.csc_matrix((np.ones(2 * nf, bool), ends.T.ravel(), np.arange(0, 2 * nf + 1, 2)), shape=(xy.shape[1], nf))
    g = Grid(2, nodes, fn, sps.csc_matrix((cf_vals, (cf_rows, cf_cols)), shape=(nf, nc)), name="Polygons")
    d = xy[:, ends[1]] - xy[:, ends[0]]
    fnorm = np.vstack((d[1], -d[0], np.zeros(nf)))
    fcent = np.vstack(((xy[:, ends[0]] + xy[:, ends[1]]) / 2, np.zeros(nf)))
    area, cc = np.zeros(nc), np.zeros((3, nc))
    for c, lp in enumerate(loops):
        x, y = xy[0, lp], xy[1, lp]
        x1, y1 = np.roll(x, -1), np.roll(y, -1)
        cr = x * y1 - x1 * y
        area[c] = cr.sum() / 2
        cc[:2, c] = ((x + x1) @ cr, (y + y1) @ cr) / (6 * area[c])
    g.set_geometry(fnorm, fcent, np.linalg.norm(d, axis=0), cc, area)
    return g


def star_polygons(ns, seed=0):
    """Irregular star-shaped polygons of ``ns`` faces (jittered angles, radii in [0.5, 1), a shear), side by side."""
    rng = np.random.default_rng(seed)
    pts, loops, start = [], [], 0
    for k, n in enumerate(ns):
        t = 2 * np.pi * (np.arange(n) + 0.8 * rng.random(n)) / n
        r = 0.5 + 0.5 * rng.random(n)
        xy = np.array([[1.0, 0.4], [0.0, 0.7]]) @ np.vstack((r * np.cos(t), r * np.sin(t))) + [[3.0 * k], [0.5 * k]]
        pts.append(xy)
        loops.append(start + np.arange(n))
        start += n
    return polygon_grid(loops, np.hstack(pts))


def anisotropic(nc, seed=1):
    """A full SPD tensor per cell of 10^3 contrast (the kzz = 1 of a 2-D tensor)."""
    rng = np.random.default_rng(seed)
    a = np.eye(2)[:, :, None] + 0.4 * rng.standard_normal((2, 2, nc))
    k = np.einsum("ikc,jkc->ijc", a, a) * 10.0 ** (3 * rng.random(nc))
    return pb.SecondOrderTensor(kxx=k[0, 0], kyy=k[1, 1], kxy=k[0, 1])


def sweep_data(g, seed=2):
    """Dirichlet on every third face, Neumann on the rest, seeded values, source and aperture."""
    rng = np.random.default_rng(seed)
    bf = np.arange(g.num_faces)
    bc = pb.BoundaryCondition(g, bf, ["dir" if f % 3 == 0 else "neu" for f in bf])
    return pb.initialize_data({}, "flow", {"second_order_tensor": anisotropic(g.num_cells), "bc": bc,
                                           "bc_values": rng.standard_normal(g.num_faces),
                                           "source": rng.standard_normal(g.num_cells),
                                           "aperture": 0.5 + rng.random(g.num_cells),
                                           "vector_source": np.zeros(3 * g.num_cells)})


@pytest.fixture
def host_build(monkeypatch):
    monkeypatch.setattr(fv, "DualGrid", EmuHybridDualGrid)


@pytest.mark.parametrize("n", SWEEP + [40, 64])
def test_mvem_on_one_polygon(n, host_build):
    """``MVEM.discretize``: the mass matrix of one n-gon against mpmath (dual_kernel has no face-count cap)."""
    g = star_polygons([n], seed=n)
    data = sweep_data(g)
    pb.MVEM("flow").discretize(g, data)
    geo, perm, rot = dual_inputs(g, data[pb.PARAMETERS]["flow"]["second_order_tensor"].values)
    M, Ms, _, _ = D.mass_reference(g, 0, geo, perm, rot)
    got = data[pb.DISCRETIZATION_MATRICES]["flow"]["mass"].toarray()
    r, at = D.worst(got, M, Ms)
    assert r <= D.MASS_TOL, (n, r, at)


@pytest.mark.parametrize("n", SWEEP)
def test_hybridization_on_one_polygon(n, host_build):
    """``HybridDualVEM.matrix_rhs``: H and its right-hand side of one n-gon against mpmath."""
    g = star_polygons([n], seed=n)
    data = sweep_data(g)
    H, rhs = pb.HybridDualVEM("flow").matrix_rhs(g, data)
    R = D.HybridReference(g, *hybrid_inputs(g, data))
    r, at = D.worst(H.toarray(), R.H, R.Hs)
    assert r <= D.HYBRID_TOL, (n, "H", r, at)
    r, at = D.worst(rhs, R.rhs, R.rs)
    assert r <= D.HYBRID_TOL, (n, "rhs", r, at)


@pytest.mark.gpu
def test_device_mixes_every_face_count_in_one_launch():
    """One grid of all polygons of 3 to 32 faces: four consecutive cells, of four sizes, share one block of
    hybrid_cell_kernel and its 32-face shared-memory layout (68,608 bytes)."""
    g = star_polygons(SWEEP, seed=5)
    check_mass(fv.DualGrid(g), g, 0, anisotropic(g.num_cells).values)
    check_hybrid(fv.DualGrid(g), g, sweep_data(g))


@pytest.mark.gpu
def test_device_mvem_above_the_hybridization_limit():
    g = star_polygons([40, 64], seed=6)
    check_mass(fv.DualGrid(g), g, 0, anisotropic(g.num_cells).values)
    with pytest.raises(NotImplementedError, match="64 faces"):
        pb.HybridDualVEM("flow").matrix_rhs(g, sweep_data(g))


def two_130gons():
    """Two circular segments of 130 edges mirrored about their common chord: the mass row of that edge gathers the
    260 faces of its two cells."""
    beta = 0.3
    th = beta + np.arange(130) * (2 * np.pi - 2 * beta) / 129     # chord ends at th[0] and th[129]
    left = np.vstack((np.cos(th) - np.cos(beta), np.sin(th)))
    left[0, [0, 129]] = 0.0
    xy = np.hstack((left, left[:, 1:129] * [[-1.0], [1.0]]))
    return polygon_grid([np.arange(130), np.r_[0, 130 + np.arange(128), 129][::-1]], xy)


@pytest.mark.gpu
def test_device_refuses_a_mass_row_of_more_than_256_faces():
    g = two_130gons()
    assert sorted(np.diff(sps.csc_matrix(g.cell_faces).indptr)) == [130, 130]
    with pytest.raises(NotImplementedError, match="more than 256 faces"):
        pb.MVEM("flow").discretize(g, sweep_data(g))


# ------------------------------------------------------------------------------------------------------------------
# non-convex polyhedra: the geometry's refusal
# ------------------------------------------------------------------------------------------------------------------


def nonconvex(kind):
    """Agglomerated hexahedra of one layer: ``L`` (3 x 2 minus a corner) and ``U`` (3 x 2 minus the middle of the top
    row), each with the left-out cell as a second cell; ``both``: a 3 x 4 layer of a cube, the L, a cube, the U and a
    cube, in that order."""
    if kind == "L":
        return agglomerate(cart_grid_3d([3, 2, 1]), np.array([0, 0, 0, 0, 1, 1]), grid_cls=Grid)
    if kind == "U":
        return agglomerate(cart_grid_3d([3, 2, 1]), np.array([0, 0, 0, 0, 1, 0]), grid_cls=Grid)
    # rows j = 0, 1: U with the notch (1, 1); rows j = 2, 3: L with (1, 3) and (2, 3) left out
    return agglomerate(cart_grid_3d([3, 4, 1]), np.array([3, 3, 3, 3, 0, 3, 1, 1, 1, 1, 2, 4]), grid_cls=Grid)


@pytest.mark.parametrize("kind", ["L", "U", "both"])
def test_host_build_refuses_nonconvex_polyhedra(kind):
    import emu_binding as eb
    with pytest.raises(ValueError, match="Some tetrahedra have negative volume"):
        eb.geometry_3d(nonconvex(kind))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["L", "U", "both"])
def test_device_refuses_nonconvex_polyhedra(kind):
    # the error names the smallest offending cell: the L (cell 0 of its grid; cell 1 of "both")
    cell = 1 if kind == "both" else 0
    with pytest.raises(ValueError, match=rf"Some tetrahedra have negative volume \(cell {cell}\)"):
        pb.compute_geometry(nonconvex(kind), assign=False)
