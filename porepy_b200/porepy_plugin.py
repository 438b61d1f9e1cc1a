"""Drop-in plugin for an installed PorePy: subclasses of ``pp.Mpfa / pp.Mpsa / pp.Biot / pp.Tpsa`` and of
the AD wrappers ``pp.ad.MpfaAd / MpsaAd / BiotAd / TpsaAd`` whose ``discretize`` runs on the GPU.

Why subclasses: ``MpfaAd.__init__`` hard-codes ``pp.Mpfa(keyword)`` (reference
src/porepy/numerics/ad/discretizations.py:192-206) and the model mixins test
``isinstance(x, pp.ad.MpfaAd)`` / ``(MpsaAd, BiotAd)`` (models/constitutive_laws.py:1341,1457,
2903), so the cores must be ``pp.Mpfa`` etc. and the wrappers ``pp.ad.MpfaAd`` etc.
``uniquify_discretization_list`` keys on ``(discr._discr.__class__, keyword)``
(numerics/ad/ad_utils.py:244-276), which stays unique for the subclasses.

Use in a model (the mixin override of constitutive_laws.py:1078,3003,3506)::

    import porepy as pp
    from porepy_b200.porepy_plugin import plugin
    b200 = plugin(pp)

    class B200Flow(pp.SinglePhaseFlow):
        def darcy_flux_discretization(self, subdomains):
            return b200.MpfaAd(self.darcy_keyword, subdomains)

    class B200Poromechanics(b200.ModelMixin, pp.Poromechanics):   # all hooks at once
        pass

    b200.install()        # or: rebind pp.Mpfa / pp.Mpsa / pp.Biot, stock models unchanged

Scope: every subdomain of a mixed-dimensional grid runs through porepy_b200 -- 3-D and 2-D grids through
the interaction-region kernels (fracture planes embedded in 3-D are rotated into their plane on the host),
1-D intersection lines through the per-face TPFA kernel (the reference's own delegation, mpfa.py:690-712,
mpsa.py:666-697), 0-D points get the empty matrices of tpfa.py:87-104.

There is NO silent CPU fallback: what the GPU classes refuse (``NotImplementedError``: periodic faces,
sub-face boundary conditions, ...) propagates to the caller.  ``plugin(pp, allow_reference_fallback=True)``
opts into handing such calls to the reference's own implementation; every such call is logged and counted
in ``b200.fallback_calls`` (GPU calls in ``b200.gpu_calls``) so that tests can assert the count is zero.
"""
from __future__ import annotations

import logging
from types import SimpleNamespace

from . import fv

logger = logging.getLogger(__name__)


def plugin(pp, allow_reference_fallback: bool = False) -> SimpleNamespace:
    """Build the plugin classes against the given ``porepy`` module."""
    fallback_calls: dict = {}
    gpu_calls: dict = {}

    def _count(d, name):
        d[name] = d.get(name, 0) + 1
    # the reference classes as they are NOW: the plugin keeps working if the caller afterwards rebinds
    # pp.Mpfa etc. to the plugin classes (e.g. to run the reference's own tests on them)
    RefMpfa, RefMpsa, RefBiot = pp.Mpfa, pp.Mpsa, pp.Biot
    RefTpfa, RefUpwind = pp.Tpfa, pp.Upwind
    RefTpsa, RefTpsaAd = pp.Tpsa, pp.ad.TpsaAd
    RefUpwindCoupling = pp.UpwindCoupling
    RefMVEM, RefRT0 = pp.MVEM, pp.RT0
    import importlib
    hybrid_module = importlib.import_module(pp.__name__ + ".numerics.vem.hybrid")
    RefHybridDualVEM = hybrid_module.HybridDualVEM
    RefMpfaAd, RefMpsaAd, RefBiotAd = pp.ad.MpfaAd, pp.ad.MpsaAd, pp.ad.BiotAd

    def _core(name, gpu_cls, ref_cls, flow):
        """Subclass of the reference core whose ``discretize`` runs on the GPU.  What the GPU classes
        refuse (``NotImplementedError``) is re-raised unless the plugin was built with
        ``allow_reference_fallback=True``."""

        if name == "Biot":  # biot.py:77 has a default keyword, the others do not
            def __init__(self, keyword: str = "mechanics") -> None:
                ref_cls.__init__(self, keyword)
                gpu_cls.__init__(self, keyword)
        else:
            def __init__(self, keyword: str) -> None:
                ref_cls.__init__(self, keyword)
                gpu_cls.__init__(self, keyword)

        def discretize(self, sd, data) -> None:
            try:
                gpu_cls.discretize(self, sd, data)
                _count(gpu_calls, name)
                return
            except NotImplementedError as e:
                if not allow_reference_fallback:
                    raise
                logger.warning("porepy_b200 %s: %s -> reference path (allow_reference_fallback)", name, e)
                _count(fallback_calls, f"{name}: {e}")
            ref_cls.discretize(self, sd, data)

        def update_discretization(self, sd, data) -> None:
            # the reference's update (index maps after a grid change, modified cells;
            # discretization.py:54-105) is host-side bookkeeping around discretize(): keep it when the
            # caller provides that information, otherwise re-discretize (on the GPU)
            if "update_discretization" in data:
                ref_cls.update_discretization(self, sd, data)
            else:
                self.discretize(sd, data)

        body = {"__init__": __init__, "discretize": discretize, "update_discretization": update_discretization,
                "__doc__": f"pp.{name} with the GPU discretization (porepy_b200.fv.{name})."}
        if name in ("MVEM", "RT0"):   # the device system while the matrices are resident, else the host formulas
            body["assemble_matrix_rhs"] = lambda self, sd, data: gpu_cls.assemble_matrix_rhs(self, sd, data)
        elif name != "Biot":
            body["assemble_matrix_rhs"] = lambda self, sd, data: ref_cls.assemble_matrix_rhs(self, sd, data)
        return type(name, (gpu_cls, ref_cls), body)

    Mpfa = _core("Mpfa", fv.Mpfa, RefMpfa, True)
    Tpfa = _core("Tpfa", fv.Tpfa, RefTpfa, False)
    Mpsa = _core("Mpsa", fv.Mpsa, RefMpsa, False)
    Biot = _core("Biot", fv.Biot, RefBiot, False)
    Tpsa = _core("Tpsa", fv.Tpsa, RefTpsa, False)
    MVEM = _core("MVEM", fv.MVEM, RefMVEM, True)
    RT0 = _core("RT0", fv.RT0, RefRT0, True)

    class Upwind(fv.Upwind, RefUpwind):
        """pp.Upwind with the per-face GPU kernel (grids of any dimension)."""

        def __init__(self, keyword: str = "transport") -> None:
            RefUpwind.__init__(self, keyword)
            fv.Upwind.__init__(self, keyword)

        def discretize(self, sd, data) -> None:
            try:
                fv.Upwind.discretize(self, sd, data)
                _count(gpu_calls, "Upwind")
                return
            except NotImplementedError as e:
                if not allow_reference_fallback:
                    raise
                logger.warning("porepy_b200 Upwind: %s -> reference path (allow_reference_fallback)", e)
                _count(fallback_calls, f"Upwind: {e}")
            RefUpwind.discretize(self, sd, data)

        def assemble_matrix_rhs(self, sd, data):
            return RefUpwind.assemble_matrix_rhs(self, sd, data)

    class HybridDualVEM(fv.HybridDualVEM, RefHybridDualVEM):
        """porepy.numerics.vem.hybrid.HybridDualVEM with the condensation and recovery on the GPU
        (porepy_b200.fv.HybridDualVEM)."""

        def __init__(self, keyword: str = "flow") -> None:
            RefHybridDualVEM.__init__(self, keyword)
            fv.HybridDualVEM.__init__(self, keyword)

        def matrix_rhs(self, g, data):
            out = fv.HybridDualVEM.matrix_rhs(self, g, data)
            _count(gpu_calls, "HybridDualVEM")
            return out

        def compute_up(self, g, solution, data):
            return fv.HybridDualVEM.compute_up(self, g, solution, data)

    class UpwindCoupling(fv.UpwindCoupling, RefUpwindCoupling):
        """pp.UpwindCoupling with the interface masks computed by the per-entry GPU kernel."""

        def __init__(self, keyword: str) -> None:
            RefUpwindCoupling.__init__(self, keyword)
            fv.UpwindCoupling.__init__(self, keyword)

        def discretize(self, sd_primary, sd_secondary, intf, data_primary, data_secondary, data_intf) -> None:
            fv.UpwindCoupling.discretize(self, sd_primary, sd_secondary, intf, data_primary, data_secondary, data_intf)
            _count(gpu_calls, "UpwindCoupling")

    def _rewrap(obj, discr, subdomains, coupling_terms=None):
        obj._discretization = discr
        if coupling_terms is None:
            pp.ad.wrap_discretization(obj, discr, subdomains=subdomains)
        else:
            pp.ad.wrap_discretization(obj=obj, discr=discr, subdomains=subdomains,
                                      coupling_terms=coupling_terms)

    class MpfaAd(RefMpfaAd):
        def __init__(self, keyword, subdomains):
            super().__init__(keyword, subdomains)
            _rewrap(self, Mpfa(keyword), subdomains)

    class MpsaAd(RefMpsaAd):
        def __init__(self, keyword, subdomains):
            super().__init__(keyword, subdomains)
            _rewrap(self, Mpsa(keyword), subdomains)

    class BiotAd(RefBiotAd):
        def __init__(self, keyword, subdomains):
            super().__init__(keyword, subdomains)
            _rewrap(self, Biot(keyword), subdomains,
                    ["displacement_divergence", "bound_displacement_divergence", "scalar_gradient",
                     "bound_pressure", "consistency"])

    class TpsaAd(RefTpsaAd):
        def __init__(self, keyword, subdomains):
            super().__init__(keyword, subdomains)
            _rewrap(self, Tpsa(keyword), subdomains)

    class ModelMixin:
        """Put FIRST among the bases of a PorePy model class to route its flux / stress
        discretizations through the GPU classes::

            class Model(b200.ModelMixin, Geometry, BoundaryConditions, pp.Poromechanics): ...

        Overrides the constitutive-law hooks (models/constitutive_laws.py:1078, 2425, 3003, 3506)
        and relaxes the exact-type check of ``add_nonlinear_diffusive_flux_discretization``
        (models/solution_strategy.py:505-524: ``type(x) in [pp.Mpfa, pp.Tpfa]``) to ``isinstance``,
        which the plugin's subclasses satisfy."""

        def darcy_flux_discretization(self, subdomains):
            return MpfaAd(self.darcy_keyword, subdomains)

        def fourier_flux_discretization(self, subdomains):
            return MpfaAd(self.fourier_keyword, subdomains)

        def stress_discretization(self, subdomains):
            stock = super().stress_discretization(subdomains)
            if isinstance(stock, RefTpsaAd):   # the TPSA models (models/momentum_balance.py:998)
                return TpsaAd(self.stress_keyword, subdomains)
            cls = BiotAd if isinstance(stock, RefBiotAd) else MpsaAd
            return cls(self.stress_keyword, subdomains)

        def add_nonlinear_diffusive_flux_discretization(self, discretization) -> None:
            if not isinstance(discretization._discr, (RefMpfa, pp.Tpfa)):
                raise TypeError(f"Expecting an Mpfa or Tpfa discretization, got {type(discretization._discr)}")
            if discretization not in self._nonlinear_diffusive_flux_discretizations:
                self._nonlinear_diffusive_flux_discretizations.append(discretization)

    def install() -> None:
        """Rebind ``pp.Mpfa / pp.Mpsa / pp.Biot`` (and ``pp.Tpfa / pp.Upwind / pp.UpwindCoupling / pp.Tpsa``) to
        the plugin classes for the whole process.  The AD
        wrappers look the cores up at construction time (``pp.Mpfa(keyword)``,
        numerics/ad/discretizations.py:192-206) and the models' exact-type checks compare with
        ``pp.Mpfa``, so every stock model then discretizes through porepy_b200 without any change to
        the model classes (this is how tools/run_reference_tests.py runs the reference's own tests)."""
        pp.Mpfa, pp.Mpsa, pp.Biot = Mpfa, Mpsa, Biot
        pp.Tpfa, pp.Upwind = Tpfa, Upwind
        pp.UpwindCoupling = UpwindCoupling
        pp.Tpsa = Tpsa
        pp.MVEM, pp.RT0 = MVEM, RT0
        hybrid_module.HybridDualVEM = HybridDualVEM

    def uninstall() -> None:
        pp.Mpfa, pp.Mpsa, pp.Biot = RefMpfa, RefMpsa, RefBiot
        pp.Tpfa, pp.Upwind = RefTpfa, RefUpwind
        pp.UpwindCoupling = RefUpwindCoupling
        pp.Tpsa = RefTpsa
        pp.MVEM, pp.RT0 = RefMVEM, RefRT0
        hybrid_module.HybridDualVEM = RefHybridDualVEM

    def md_flow_from_model(model, keyword=None):
        """The mixed-dimensional Darcy problem of a prepared single-phase flow model (``pp.SinglePhaseFlow`` after
        ``prepare_simulation``) as a ``porepy_b200.mdflow.MixedDimensionalFlow``: grids, parameter dictionaries and
        mortar projections of ``model.mdg`` as they are, boundary data, normal permeability, apertures and specific
        volumes evaluated from the model's own constitutive laws (models/constitutive_laws.py:203-282, 1032-1076).
        ``.discretize()`` then runs ``porepy_b200.Mpfa`` on every subdomain and ``.assemble()`` / ``.solve()`` build and
        solve the coupled Jacobian on the device -- with unit mobility (the model's Jacobian is then state independent)
        it equals ``model.equation_system.assemble()``."""
        import numpy as np
        from .mdflow import MixedDimensionalFlow
        mdg = model.mdg
        kw = keyword or model.darcy_keyword

        def evaluated(op, n):
            v = model.equation_system.evaluate(op)
            return np.full(n, float(v)) if np.ndim(v) == 0 else np.asarray(v, float)

        def bc_values(sd):
            bg = mdg.subdomain_to_boundary_grid(sd)
            if bg is None or bg.num_cells == 0:
                return np.zeros(sd.num_faces)
            bc = mdg.subdomain_data(sd)[pp.PARAMETERS][kw]["bc"]
            proj = bg.projection()
            return np.where(bc.is_dir, proj.T @ model.bc_values_pressure(bg), proj.T @ model.bc_values_darcy_flux(bg))
        return MixedDimensionalFlow.from_mdg(
            mdg, kw, bc_values=bc_values,
            normal_permeability=lambda it: evaluated(model.normal_permeability([it]), it.num_cells),
            aperture=lambda sd: evaluated(model.aperture([sd]), sd.num_cells),
            specific_volume=lambda it: evaluated(model.specific_volume([it]), it.num_cells))

    from . import model_bridge as bridge
    return SimpleNamespace(Mpfa=Mpfa, Mpsa=Mpsa, Biot=Biot, Tpfa=Tpfa, Tpsa=Tpsa, MVEM=MVEM, RT0=RT0, HybridDualVEM=HybridDualVEM, Upwind=Upwind, UpwindCoupling=UpwindCoupling,
                           MpfaAd=MpfaAd, MpsaAd=MpsaAd, BiotAd=BiotAd, TpsaAd=TpsaAd,
                           ModelMixin=ModelMixin, install=install, uninstall=uninstall, md_flow_from_model=md_flow_from_model,
                           # nonlinear model problems on the device AD chain (porepy_b200/model_bridge.py)
                           compressible_flow_from_model=bridge.compressible_flow_from_model,
                           mass_energy_from_model=bridge.mass_energy_from_model,
                           poromechanics_from_model=bridge.poromechanics_from_model,
                           thermoporomechanics_from_model=bridge.thermoporomechanics_from_model,
                           fractured_momentum_from_model=bridge.fractured_momentum_from_model,
                           fractured_poromechanics_from_model=bridge.fractured_poromechanics_from_model,
                           fractured_thermoporomechanics_from_model=bridge.fractured_thermoporomechanics_from_model,
                           tpsa_momentum_from_model=bridge.tpsa_momentum_from_model,
                           tpsa_poromechanics_from_model=bridge.tpsa_poromechanics_from_model,
                           tpsa_thermoporomechanics_from_model=bridge.tpsa_thermoporomechanics_from_model,
                           tpsa_fractured_momentum_from_model=bridge.tpsa_fractured_momentum_from_model,
                           fallback_calls=fallback_calls, gpu_calls=gpu_calls)
