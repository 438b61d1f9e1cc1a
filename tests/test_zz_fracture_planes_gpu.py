"""GPU leg of tests/test_embedded_planes.py: flux discretization of fracture planes (2-D grids
embedded in 3-D, ``ambient_dimension = 3``; reference mpfa.py:733-754 / 423-466) through the real
device plan, against golden fixtures written by the reference."""
import pytest

import porepy_b200 as pb
from cases import load_case, max_rel_err
from golden_io import case_names

pytestmark = pytest.mark.gpu
TOL = 1e-10


@pytest.mark.parametrize("name", case_names("embedded_"))
def test_fracture_plane_flux_discretization(name):
    c = load_case(name)
    k = pb.SecondOrderTensor.from_values(c.raw["K"])
    data = pb.initialize_data({}, "flow", {"second_order_tensor": k, "bc": c.bc,
                                           "ambient_dimension": int(c.raw["ambient_dimension"])})
    pb.Mpfa("flow").discretize(c.g, data)
    got = data[pb.DISCRETIZATION_MATRICES]["flow"]
    assert got["vector_source"].shape == (c.g.num_faces, 3 * c.g.num_cells)
    err, key = max_rel_err(c.mats, got)
    assert err < TOL, (key, err)


@pytest.mark.parametrize("name", case_names("embedded_"))
def test_fracture_plane_device_system_with_gravity(name):
    """``assemble_matrix_rhs`` on a fracture plane with a 3-component vector source: the device path (values in the
    plane's frame, the vector rotated into it) equals the host products with the lifted matrices."""
    import numpy as np
    c = load_case(name)
    rng = np.random.default_rng(1)
    k = pb.SecondOrderTensor.from_values(c.raw["K"])
    amb = int(c.raw["ambient_dimension"])
    bv = rng.random(c.g.num_faces)
    vs = rng.standard_normal(amb * c.g.num_cells)
    data = pb.initialize_data({}, "flow", {"second_order_tensor": k, "bc": c.bc, "ambient_dimension": amb,
                                           "bc_values": bv, "vector_source": vs})
    d = pb.Mpfa("flow")
    d.discretize(c.g, data)
    A_dev, b_dev = d.assemble_matrix_rhs(c.g, data)
    assert A_dev.device_csr is not None
    div = c.g.divergence(dim=1)
    b_ref = -div @ (c.mats["bound_flux"] @ bv) - div @ (c.mats["vector_source"] @ vs)
    A_ref = div @ c.mats["flux"]
    assert abs(A_ref - A_dev).max() <= 1e-10 * abs(A_ref).max()
    assert np.abs(b_dev - b_ref).max() <= 1e-10 * np.abs(b_ref).max()
