"""The sub-cell topology plan built on the device (csrc/plan_device.cu) against the host construction
(csrc/plan_host.hpp, forced with POREB200_HOST_PLAN=1): same patterns and the same discretization matrices on
hexahedra, tetrahedra (structured and Delaunay), 2-D grids and a grid with boundary-heavy nodes, and the same
mechanics system A = div_nd @ stress assembled on the device from either plan."""
import os

import numpy as np
import pytest
import scipy.sparse as sps

import porepy_b200 as pb
from cases import flatten, load_case
from golden_io import rel_err

pytestmark = pytest.mark.gpu


def _both_plans(g, run):
    out = []
    for host in (False, True):
        if hasattr(g, "_b200_plan"):
            del g._b200_plan
        if host:
            os.environ["POREB200_HOST_PLAN"] = "1"
        try:
            out.append(run())
        finally:
            os.environ.pop("POREB200_HOST_PLAN", None)
    if hasattr(g, "_b200_plan"):
        del g._b200_plan
    return out


@pytest.mark.parametrize("name", ["mpfa_cart3d_pert", "mpfa_tet3d_delaunay", "mpfa_tri2d", "mpfa_cart2d"])
def test_device_plan_equals_host_plan_on_golden_grids(name):
    c = load_case(name)

    def run():
        plan = pb.DevicePlan.for_grid(c.g)
        pats = [tuple(np.array(a) for a in plan.base_pattern(w)) for w in range(4)]
        data = pb.initialize_data({}, "flow", {"second_order_tensor": pb.SecondOrderTensor.from_values(c.raw["K"]),
                                               "bc": c.bc, "mpfa_eta": c.eta})
        pb.Mpfa("flow").discretize(c.g, data)
        return plan.sizes(), pats, {k: m.copy() for k, m in data[pb.DISCRETIZATION_MATRICES]["flow"].items()}
    (sz_d, pat_d, m_d), (sz_h, pat_h, m_h) = _both_plans(c.g, run)
    assert sz_d == sz_h
    for (ipd, ixd), (iph, ixh) in zip(pat_d, pat_h):
        assert np.array_equal(ipd, iph) and np.array_equal(ixd, ixh)
    for key in m_h:
        assert rel_err(m_h[key], m_d[key]) < 1e-13, key
        assert rel_err(c.mats[key], m_d[key]) < 1e-10, key


@pytest.mark.parametrize("make", [lambda: pb.structured_tet_grid([7, 6, 5]), lambda: pb.cart_grid_3d([9, 8, 7], perturb=0.2)])
def test_device_plan_equals_host_plan_biot(make):
    g = make()
    rng = np.random.default_rng(5)
    nc = g.num_cells
    C = pb.FourthOrderTensor(np.exp(0.3 * rng.standard_normal(nc)), np.exp(0.3 * rng.standard_normal(nc)))
    bf = g.get_all_boundary_faces()
    vbc = pb.BoundaryConditionVectorial(g, bf[g.face_centers[2, bf] < 1e-10], "dir")

    def run():
        data = pb.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": vbc, "scalar_vector_mappings": {"p": 0.7}})
        pb.Biot("mech").discretize(g, data)
        return {k: m.copy() for k, m in flatten(data[pb.DISCRETIZATION_MATRICES]["mech"]).items()}
    m_d, m_h = _both_plans(g, run)
    for key in m_h:
        assert m_d[key].shape == m_h[key].shape
        assert rel_err(m_h[key], m_d[key]) < 1e-12, key


@pytest.mark.parametrize("make", [lambda: pb.cart_grid_3d([6, 5, 4], perturb=0.3, seed=2),
                                  lambda: pb.structured_tet_grid([4, 4, 3])])
def test_device_mechanics_system_from_host_and_device_plan(make):
    """pb_mpsa_system gathers each cell's faces through the plan's cell -> face lists, which the host-topology plan
    uploads itself: the same matrix and pattern from both plans, and the scipy product g.divergence(dim=3) @ stress."""
    g = make()
    rng = np.random.default_rng(11)
    nc = g.num_cells
    C = pb.FourthOrderTensor(np.exp(0.4 * rng.standard_normal(nc)), np.exp(0.4 * rng.standard_normal(nc)))
    bf = g.get_all_boundary_faces()
    vbc = pb.BoundaryConditionVectorial(g, bf[g.face_centers[2, bf] < 1e-10], "dir")

    def run():
        data = pb.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": vbc,
                                               "bc_values": np.zeros(3 * g.num_faces), "source": np.zeros(3 * nc)})
        d = pb.Mpsa("mech")
        d.discretize(g, data)
        a_dev, _ = d.assemble_matrix_rhs_device(g, data)
        stress = sps.csr_matrix(data[pb.DISCRETIZATION_MATRICES]["mech"]["stress"])
        return a_dev.to_scipy(), (g.divergence(dim=3) @ stress).tocsr()
    (a_d, ref_d), (a_h, ref_h) = _both_plans(g, run)
    assert a_d.shape == a_h.shape == (3 * nc, 3 * nc)
    assert np.array_equal(a_d.indptr, a_h.indptr) and np.array_equal(a_d.indices, a_h.indices)
    assert rel_err(a_d, a_h) < 1e-13
    assert rel_err(ref_d, a_d) < 1e-13
    assert rel_err(ref_h, a_h) < 1e-13
