"""The upwinded advective terms of the model classes: re-discretization of ``porepy_b200.Upwind`` /
``UpwindCoupling`` from the iterate's Darcy flux (the reference's ``before_nonlinear_iteration``,
models/solution_strategy.py:433-441) and the advective flux q (U w) + B_dir (q w_b) + B_neu w_n
(constitutive_laws.py:2521-2569) on the device AD chain."""
from __future__ import annotations

from types import SimpleNamespace

from . import ad
from .fv import Upwind, UpwindCoupling
from .params import PARAMETERS


def rediscretize_upwind(sd, data, keyword: str, darcy_flux, bc) -> None:
    """``Upwind(keyword)`` on ``sd`` from the face fluxes ``darcy_flux`` (host array) and the boundary condition ``bc``."""
    prm = data.setdefault(PARAMETERS, {}).setdefault(keyword, {})
    prm["darcy_flux"], prm["bc"] = darcy_flux, bc
    Upwind(keyword).discretize(sd, data)


def rediscretize_upwind_coupling(sd_primary, sd_secondary, num_mortar_cells: int, data_primary, data_secondary,
                                 intf_data, keyword: str, darcy_flux) -> None:
    """``UpwindCoupling(keyword)`` on an interface from the mortar fluxes ``darcy_flux`` (host array)."""
    intf_data.setdefault(PARAMETERS, {}).setdefault(keyword, {})["darcy_flux"] = darcy_flux
    UpwindCoupling(keyword).discretize(sd_primary, sd_secondary, SimpleNamespace(num_cells=num_mortar_cells),
                                       data_primary, data_secondary, intf_data)


def advective_flux(matrices, flux, weight, dirichlet=None, neumann=None):
    """flux (transport weight) + rhs_dir (flux dirichlet) + rhs_neu neumann, with ``matrices`` the ``Upwind``
    discretization.  A boundary term is added only when its values are given: leaving it out keeps a zero term out of
    the Jacobian's pattern."""
    csr = ad.as_device_csr
    out = flux * (csr(matrices["transport"]) @ weight)
    if dirichlet is not None:
        out = out + (csr(matrices["rhs_dir"]) @ (flux * dirichlet))
    if neumann is not None:
        out = out + (csr(matrices["rhs_neu"]) @ neumann)
    return out
