"""Frictional contact on a fracture (the contact part of BASELINE config[4]): the reference's ``pp.MomentumBalance`` --
MPSA in the matrix, interface force balance, the semismooth normal / tangential complementarity laws with Coulomb friction
and shear dilation -- on the device AD chain (porepy_b200/contact.py) against the unmodified reference: Jacobian and residual
at the second Newton iterate, the residual history of the semismooth Newton loop and the converged SLIDING state
(tests/golden/contact_model.npz, tools/make_contact_golden.py).
CPU: host build of the node routines + the scipy stand-in for the device sparse algebra."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sps
import scipy.sparse.linalg as spla

import porepy_b200 as pb
from porepy_b200.contact import FractureContact, FracturedMomentumBalance
from porepy_b200.grid import Grid
from golden_io import GOLDEN_DIR


def _csr(d, key):
    return sps.csr_matrix((d[key + "__data"], d[key + "__indices"], d[key + "__indptr"]), shape=tuple(d[key + "__shape"]))


CASES = ["contact_model", "contact_sticking", "contact_open", "contact_mixed"]   # sliding / sticking / open / open + sliding


def load_problem(name="contact_model"):
    d = dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False))
    g = Grid.from_arrays({k[len("matrix__"):]: v for k, v in d.items() if k.startswith("matrix__")})
    nf = g.num_faces
    vbc = SimpleNamespace(is_dir=d["mech_is_dir"], is_neu=d["mech_is_neu"], is_rob=d["mech_is_rob"],
                          is_internal=d["mech_is_internal"], robin_weight=np.zeros((3, 3, nf)), bc_type="vectorial",
                          num_faces=nf)
    data = pb.initialize_data({}, "mechanics", {"fourth_order_tensor": pb.FourthOrderTensor.from_values(d["C"]), "bc": vbc})
    frac = FractureContact(_csr(d, "mortar_to_primary_avg"), _csr(d, "primary_to_mortar_int"),
                           _csr(d, "mortar_to_secondary_avg"), _csr(d, "secondary_to_mortar_int"), d["mortar_sign"],
                           d["mortar_volumes"], _csr(d, "local_coordinates"))
    constants = {k: float(d[k]) for k in ("numerical_constant", "characteristic_traction", "friction_coefficient",
                                          "dilation_angle", "reference_gap", "open_state_tolerance")}
    return FracturedMomentumBalance(g, data, d["mech_bc_values"], [frac], constants), d


def check(prob, d, to_host, make_tensor):
    cm = d["column_map"]
    assert np.array_equal(cm, np.arange(prob.num_dofs))            # one fracture: the reference's order is [u | t | u_j]
    J, rhs = prob.linearize(d["iterate"], d["previous"])
    Jref, bref = _csr(d, "iterate_jacobian"), d["iterate_rhs"]
    assert abs(J.to_scipy() - Jref).max() <= 1e-10 * abs(Jref).max()
    # (in the sticking and open cases the stored iterate is already converged: compare on the Jacobian's scale then)
    assert np.abs(to_host(rhs) - bref).max() <= 1e-10 * max(np.abs(bref).max(), 1e-3 * abs(Jref).max())

    def direct(Jd, r):                                             # zeros on the diagonal of the complementarity rows
        return make_tensor(spla.spsolve(Jd.to_scipy().tocsc(), to_host(r)))
    x, hist = prob.time_step(d["previous"], direct, tol=1e-11)
    ref = d["residual_norms"]
    assert hist[-1]["residual"] <= 1e-10 * hist[0]["residual"] and len(hist) <= len(ref) + 1, hist
    for mine, theirs in zip(hist[:4], ref[:4]):                    # the semismooth loop's own (non-monotone) history
        if theirs > 1e-9 * ref[0]:
            assert abs(mine["residual"] - theirs) <= 0.05 * theirs, (hist, ref)
    xh = to_host(x)
    assert np.linalg.norm(xh - d["solution"]) <= 1e-8 * np.linalg.norm(d["solution"])
    # the contact conditions at the converged state: open cells carry no traction, closed ones a compressive normal
    # traction and a tangential one inside (sticking) or on (sliding) the friction cone
    t = prob.unknown_layout.parts(xh)["contact_traction"][0].reshape(-1, 3)
    mu = float(d["friction_coefficient"])
    is_open = np.abs(t[:, 2]) < 1e-12
    assert np.all(np.abs(t[is_open]) < 1e-12) and np.all(t[~is_open, 2] < 0)
    assert np.all(np.linalg.norm(t[~is_open, :2], axis=1) <= mu * np.abs(t[~is_open, 2]) * (1 + 1e-8))
    return t


@pytest.mark.parametrize("name", CASES)
def test_frictional_contact_host_build(name, monkeypatch):
    import torch
    from emu_binding import EmuBackedPlan
    from porepy_b200 import fv
    import emu_sparse
    monkeypatch.setattr(fv, "DevicePlan", EmuBackedPlan)
    emu_sparse.install(monkeypatch)
    prob, d = load_problem(name)
    prob.discretize()
    t = check(prob, d, lambda t: t.numpy(), lambda a: torch.as_tensor(np.asarray(a, float)))
    mu = float(d["friction_coefficient"])
    ratio = np.linalg.norm(t[:, :2], axis=1) / np.maximum(mu * np.abs(t[:, 2]), 1e-300)
    expect = {"contact_model": lambda: np.allclose(ratio, 1.0, rtol=1e-8),            # sliding everywhere
              "contact_sticking": lambda: np.all(ratio < 0.2),
              "contact_open": lambda: np.all(t == 0.0),
              "contact_mixed": lambda: np.sum(np.abs(t[:, 2]) < 1e-12) == 2 and np.allclose(ratio[np.abs(t[:, 2]) > 1e-12], 1.0)}
    assert expect[name](), (name, t)
