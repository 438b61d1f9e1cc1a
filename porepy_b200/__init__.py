"""porepy_b200 -- H100 (sm_90a) MPFA / MPSA / Biot interaction-region assembly and CSR
SpMV behind PorePy's ``Discretization.discretize() / assemble_matrix_rhs()`` operator API.

The CUDA library (``libporeb200.so``, built in-tree by ``porepy_b200.build``) is loaded on
first use; there is no CPU fallback.
"""
from .contact import FractureContact, FracturedMomentumBalance  # noqa: F401
from .fractured_poromech import FractureCoupling, FracturedPoromechanics  # noqa: F401
from .fractured_thm import FracturedThermoporomechanics  # noqa: F401
from .fv import (MVEM, RT0, Biot, DevicePlan, DualGrid, FaceGrid, HybridDualVEM, Mpfa, Mpsa, Tpfa, Tpsa, Upwind, UpwindCoupling,  # noqa: F401
                 determine_eta)
from .geometry import compute_geometry  # noqa: F401
from .grid import Grid, cart_grid_2d, cart_grid_3d, structured_tet_grid, tet_grid_from_cells  # noqa: F401
from .mdflow import MdInterface, MdSubdomain, MixedDimensionalFlow  # noqa: F401
from .mdflow_nl import CompressibleMixedDimensionalFlow  # noqa: F401
from .mdthermal import MixedDimensionalMassEnergy  # noqa: F401
from .poromech import Poromechanics  # noqa: F401
from .params import (DISCRETIZATION_MATRICES, PARAMETERS, BoundaryCondition,  # noqa: F401
                     BoundaryConditionVectorial, FourthOrderTensor, SecondOrderTensor,
                     initialize_data)
from .sparse import DeviceCsr  # noqa: F401
from .thermoporomech import Thermoporomechanics  # noqa: F401
from .tpsa_elasticity import TpsaElasticity  # noqa: F401
from .tpsa_poromech import TpsaPoromechanics  # noqa: F401
from .tpsa_thermoporomech import TpsaThermoporomechanics  # noqa: F401
from .tpsa_contact import TpsaFracturedMomentumBalance  # noqa: F401
from .tpfa_ad import DifferentiableTpfa  # noqa: F401

__all__ = ["Mpfa", "Mpsa", "Biot", "Tpfa", "Tpsa", "MVEM", "RT0", "HybridDualVEM", "DualGrid", "Upwind", "UpwindCoupling", "DevicePlan", "FaceGrid", "DeviceCsr", "Grid", "cart_grid_2d", "cart_grid_3d",
           "structured_tet_grid", "tet_grid_from_cells", "SecondOrderTensor", "FourthOrderTensor",
           "BoundaryCondition", "BoundaryConditionVectorial", "initialize_data", "PARAMETERS",
           "DISCRETIZATION_MATRICES", "determine_eta", "compute_geometry", "DifferentiableTpfa",
           "MixedDimensionalFlow", "MdSubdomain", "MdInterface", "CompressibleMixedDimensionalFlow", "Poromechanics", "Thermoporomechanics", "MixedDimensionalMassEnergy", "FracturedMomentumBalance", "FractureContact", "FracturedPoromechanics", "FractureCoupling", "FracturedThermoporomechanics", "TpsaElasticity", "TpsaPoromechanics", "TpsaThermoporomechanics", "TpsaFracturedMomentumBalance"]
