"""Two-point stress approximation (``porepy_b200.Tpsa``, csrc/tpsa_face.cuh) against the unmodified reference's
``pp.Tpsa.discretize``: the golden fixtures of tools/make_tpsa_golden.py on the host build of the per-face routine and
on the GPU, the reference's refusals, whole TPSA models through the PorePy plugin, and the bench-size mesh on the GPU
against the reference run from oracle/_ref."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sps

import porepy_b200 as pb
from porepy_b200 import fv
from golden_io import case_names, load_case, rel_err
from tpsa_checks import full_size_mechanics, use_host_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from ref_loader import load_porepy, reference_available  # noqa: E402

CASES = case_names("tpsa_")
KEYS = ("stress", "stress_rotation", "stress_total_pressure", "rotation_displacement", "rotation_rotation",
        "solid_mass_displacement", "solid_mass_total_pressure", "bound_displacement_cell",
        "bound_displacement_rotation_cell", "bound_displacement_solid_pressure_cell", "bound_stress",
        "bound_rotation_displacement", "bound_mass_displacement", "bound_displacement_face")
TOL = 1e-12


@pytest.fixture()
def host_build(monkeypatch):
    use_host_build(monkeypatch, plan=False, sparse=False)


def _discretize(c):
    c.g.tags["fracture_faces"] = np.asarray(c.raw["fracture_faces"], bool)
    bmask = np.zeros(c.g.num_faces, bool)
    bmask[c.g.get_all_boundary_faces()] = True
    assert np.array_equal(bmask, c.raw["boundary_faces"])
    C = pb.FourthOrderTensor(c.raw["mu"], np.ones(c.g.num_cells))
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": c.bc})
    pb.Tpsa("mech").discretize(c.g, data)
    return data[pb.DISCRETIZATION_MATRICES]["mech"]


def _assert_matches(ref: dict, got: dict, tol=TOL):
    assert set(KEYS) <= set(got)
    for key in KEYS:
        r, m = sps.csr_matrix(ref[key]), sps.csr_matrix(got[key])
        assert r.shape == m.shape, (key, r.shape, m.shape)
        if r.nnz == 0 or abs(r).max() == 0:   # e.g. rotation_rotation with Dirichlet conditions only
            d = abs(r - m)
            assert (d.max() if d.nnz else 0.0) <= tol, key
        else:
            assert rel_err(r, m) <= tol, (key, rel_err(r, m))


def test_fixtures_present():
    assert len(CASES) >= 7, CASES


@pytest.mark.parametrize("name", CASES)
def test_host_build_matches_reference(name, host_build):
    c = load_case(name)
    _assert_matches(c.mats, _discretize(c))


def _grid_2d():
    g = pb.cart_grid_2d([3, 2])
    return g


def _params(g, bc=None):
    if bc is None:
        bf = g.get_all_boundary_faces()
        bc = pb.BoundaryConditionVectorial(g, bf, "dir")
    C = pb.FourthOrderTensor(np.ones(g.num_cells), np.ones(g.num_cells))
    return pb.initialize_data({}, "mech", {"fourth_order_tensor": C, "bc": bc})


def test_refusals_and_messages(host_build):
    g = _grid_2d()
    bf = g.get_all_boundary_faces()
    bc = pb.BoundaryConditionVectorial(g, bf, "dir")
    bc.basis = bc.basis.copy()
    bc.basis[0, 1, bf[0]] = 0.5
    with pytest.raises(NotImplementedError, match="Have not implemented Robin conditions with a non-trivial basis."):
        pb.Tpsa("mech").discretize(g, _params(g, bc))
    bc = pb.BoundaryConditionVectorial(g, bf, "rob")
    bc.robin_weight = bc.robin_weight.copy()
    bc.robin_weight[1, 0, bf[1]] = 0.3
    with pytest.raises(NotImplementedError, match="Non-diagonal Robin weights have not been implemnted."):
        pb.Tpsa("mech").discretize(g, _params(g, bc))
    bc = pb.BoundaryConditionVectorial(g, bf, "rob")
    bc.is_rob[1, bf[2]] = False
    bc.is_dir[1, bf[2]] = True
    with pytest.raises(NotImplementedError, match="Mixing Robin with Dirichlet or Neumann"):
        pb.Tpsa("mech").discretize(g, _params(g, bc))
    g3 = pb.cart_grid_3d([2, 2, 2])
    g3.periodic_face_map = np.zeros((2, 0), int)
    with pytest.raises(NotImplementedError, match="periodic"):
        pb.Tpsa("mech").discretize(g3, _params(g3))
    line = type("Line", (), {"dim": 1, "num_cells": 2, "num_faces": 3})()
    with pytest.raises(NotImplementedError, match="Tpsa is only implemented for 2d and 3d grids."):
        pb.Tpsa("mech").discretize(line, {pb.PARAMETERS: {"mech": {}}})
    with pytest.raises(NotImplementedError, match="Tpsa is only implemented for 2d and 3d grids."):
        pb.Tpsa("mech").ndof(line)
    with pytest.raises(NotImplementedError, match="cannot be used for assembly"):
        pb.Tpsa("mech").assemble_matrix_rhs(g, _params(g))


def test_ndof_and_keys():
    g2, g3 = pb.cart_grid_2d([3, 2]), pb.cart_grid_3d([2, 2, 2])
    assert pb.Tpsa("m").ndof(g2) == 4 * g2.num_cells
    assert pb.Tpsa("m").ndof(g3) == 7 * g3.num_cells
    t = pb.Tpsa("m")
    assert sorted(t._term_keys()) == sorted(KEYS)
    if not reference_available():
        return
    pp = load_porepy()
    ref = pp.Tpsa("m")
    keys = {k: v for k, v in vars(ref).items() if k.endswith("_matrix_key")}
    assert keys == {k: v for k, v in vars(t).items() if k.endswith("_matrix_key")}
    assert ref.ndof(g2) == t.ndof(g2) and ref.ndof(g3) == t.ndof(g3)


# ---- GPU ------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_gpu_matches_reference_and_host_build(name, monkeypatch):
    c = load_case(name)
    got = _discretize(c)
    _assert_matches(c.mats, got)
    with monkeypatch.context() as m:
        use_host_build(m, plan=False, sparse=False)
        host = _discretize(load_case(name))
    for key in KEYS:   # same routine, the device build contracts some products into FMAs
        a, b = host[key], got[key]
        assert np.array_equal(a.indptr, b.indptr) and np.array_equal(a.indices, b.indices), key
        scale = max(np.abs(a.data).max(initial=0.0), 1e-300)
        assert np.abs(a.data - b.data).max(initial=0.0) <= 1e-13 * scale, key


@pytest.mark.gpu
def test_gpu_refuses_bad_shear_modulus():
    g = _grid_2d()
    data = _params(g)
    data[pb.PARAMETERS]["mech"]["fourth_order_tensor"].mu[1] = 0.0
    with pytest.raises(ValueError, match="shear modulus"):
        pb.Tpsa("mech").discretize(g, data)


@pytest.mark.gpu
@pytest.mark.skipif(not reference_available(), reason="oracle/_ref not present (run oracle/make_ref.sh)")
def test_full_size_matches_reference():
    """998,250 tetrahedra (the bench mesh) with Dirichlet, roller, Robin and Neumann faces: all 14 matrices equal the
    reference's run on the same host arrays."""
    from oracle.ref_loader import reference_grid
    pp = load_porepy()
    g, bc, mu = full_size_mechanics()
    assert g.num_cells == 998_250
    data = pb.initialize_data({}, "mech", {"fourth_order_tensor": pb.FourthOrderTensor(mu, np.ones_like(mu)),
                                           "bc": bc})
    pb.Tpsa("mech").discretize(g, data)
    got = data[pb.DISCRETIZATION_MATRICES]["mech"]
    r = reference_grid(pp, g)
    rbc = pp.BoundaryConditionVectorial(r)
    rbc.is_dir, rbc.is_neu, rbc.is_rob = bc.is_dir.copy(), bc.is_neu.copy(), bc.is_rob.copy()
    rbc.robin_weight = bc.robin_weight.copy()
    rdata = pp.initialize_data({}, "mech", {"fourth_order_tensor": pp.FourthOrderTensor(mu, np.ones_like(mu)),
                                            "bc": rbc})
    pp.Tpsa("mech").discretize(r, rdata)
    _assert_matches(rdata[pp.DISCRETIZATION_MATRICES]["mech"], got)


# ---- whole TPSA models through the plugin ---------------------------------------------------------------------


class _Square:
    def set_domain(self):
        import porepy as pp
        box = {"xmin": 0, "xmax": 1, "ymin": 0, "ymax": 1}
        if self.params.get("tpsa_nd", 2) == 3:
            box.update(zmin=0, zmax=1)
        self._domain = pp.Domain(box)

    def grid_type(self):
        return "cartesian"

    def meshing_arguments(self):
        return {"cell_size": 0.25}


class _TpsaMechBC:
    def bc_type_mechanics(self, sd):
        import porepy as pp
        sides = self.domain_boundary_sides(sd)
        bc = pp.BoundaryConditionVectorial(sd, sides.west, "dir")
        bc.is_dir[1, sides.south] = True      # roller
        bc.is_neu[1, sides.south] = False
        bc.internal_to_dirichlet(sd)
        return bc

    def bc_values_stress(self, bg):
        sides = self.domain_boundary_sides(bg)
        v = np.zeros((self.nd, bg.num_cells))
        v[1, sides.north] = -1e-3 * bg.cell_volumes[sides.north]
        v[0, sides.east] = 5e-4 * bg.cell_volumes[sides.east]
        return v.ravel("F")


def _model_solve(pp, cls, nd):
    model = cls({"times_to_export": [], "tpsa_nd": nd,
                 "time_manager": pp.TimeManager([0, 1.0], 0.5, constant_dt=True)})
    pp.run_time_dependent_model(model, {"prepare_simulation": True})
    return model.equation_system.get_variable_values(iterate_index=0)


def _model_classes(pp, family):
    if family == "momentum":
        return (pp.models.momentum_balance.TpsaMomentumBalanceMixin, _Square, _TpsaMechBC, pp.MomentumBalance)
    from test_porepy_plugin import _FlowBC
    return (pp.models.poromechanics.TpsaPoromechanicsMixin, _Square, _FlowBC, _TpsaMechBC, pp.Poromechanics)


def _check_models(pp, family, nd):
    from porepy_b200.porepy_plugin import plugin
    bases = _model_classes(pp, family)

    class Stock(*bases):
        pass
    ref = _model_solve(pp, Stock, nd)
    assert np.linalg.norm(ref) > 0
    # 1) install(): the stock class, pp.Tpsa rebound
    b = plugin(pp)
    b.install()
    try:
        assert pp.Tpsa is b.Tpsa
        got = _model_solve(pp, Stock, nd)
    finally:
        b.uninstall()
    assert pp.Tpsa is not b.Tpsa
    assert b.gpu_calls.get("Tpsa", 0) >= 1 and b.fallback_calls == {}
    assert np.linalg.norm(ref - got) <= 1e-10 * np.linalg.norm(ref)
    # 2) ModelMixin: the stock TpsaAd is replaced by the plugin's (not by MpsaAd)
    b2 = plugin(pp)

    class Mixed(b2.ModelMixin, *bases):
        pass
    got2 = _model_solve(pp, Mixed, nd)
    assert b2.gpu_calls.get("Tpsa", 0) >= 1 and b2.fallback_calls == {}
    assert "Mpsa" not in b2.gpu_calls and "Biot" not in b2.gpu_calls
    assert np.linalg.norm(ref - got2) <= 1e-10 * np.linalg.norm(ref)


MODELS = [("momentum", 2), ("momentum", 3), ("poromechanics", 2)]


@pytest.mark.skipif(not reference_available(), reason="reference tree not present")
@pytest.mark.parametrize("family,nd", MODELS)
def test_models_through_the_plugin_host_build(family, nd, monkeypatch):
    from emu_binding import emu_interface_upwind_masks
    use_host_build(monkeypatch, sparse=False)
    monkeypatch.setattr(fv, "interface_upwind_masks", emu_interface_upwind_masks)
    _check_models(load_porepy(), family, nd)


@pytest.mark.gpu
@pytest.mark.skipif(not reference_available(), reason="oracle/_ref not present (run oracle/make_ref.sh)")
@pytest.mark.parametrize("family,nd", MODELS)
def test_models_through_the_plugin_gpu(family, nd):
    from porepy_b200 import _lib
    _lib.require_gpu()
    _check_models(load_porepy(), family, nd)
