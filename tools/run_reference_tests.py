"""Run the REFERENCE's own finite-volume unit tests (tests/numerics/fv/test_{mpfa,mpsa,biot,tpsa}.py of the
read-only tree) with pp.Mpfa / pp.Mpsa / pp.Biot / pp.Tpsa (and pp.Tpfa / pp.Upwind / pp.MVEM / pp.RT0 / HybridDualVEM) rebound to the
porepy_b200 plugin classes.  The mixed schemes' tests are named on the command line:

    python tools/run_reference_tests.py numerics/vem/test_dual_vem.py numerics/vem/test_rt0.py
    python tools/run_reference_tests.py numerics/vem/test_hybrid_vem.py   # HybridDualVEM.matrix_rhs counted as well

    python tools/run_reference_tests.py            # build container or any box with /root/reference
    python tools/run_reference_tests.py functional/test_terzaghi.py [--stock] [pytest options]

With a GPU the plugin runs the CUDA path; without one the device plan is replaced by the host build of the
same node routines (tests/emu) so that the drop-in wiring can be checked in the build container.  Prints
how many discretize() calls ran on the porepy_b200 path and, with the reason, every call the plugin handed
to the reference (this tool opts into ``allow_reference_fallback``; the default plugin re-raises).  Nothing is copied
from the reference; its test files are collected where they lie."""
import collections
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
REF_TESTS = "/root/reference/tests/numerics/fv"
COUNTS = collections.Counter()


class Rebind:
    """pytest plugin object: rebinding happens before collection imports the test modules."""

    def pytest_configure(self, config):
        from ref_loader import load_porepy
        pp = load_porepy()
        from porepy_b200 import _lib, fv
        from porepy_b200.porepy_plugin import plugin
        try:
            gpu = _lib.load().pb_device_count() > 0
        except Exception:
            gpu = False
        if not gpu:
            from emu_binding import EmuBackedPlan
            from emu_tpsa import EmuTpsaFaceGrid   # the host build of the per-face routines, TPSA included
            from emu_dual_hybrid import EmuHybridDualGrid   # the host build of MVEM / RT0 and their hybridization
            fv.DevicePlan = EmuBackedPlan
            fv.FaceGrid = EmuTpsaFaceGrid
            fv.DualGrid = EmuHybridDualGrid
            import emu_binding
            fv.interface_upwind_masks = emu_binding.emu_interface_upwind_masks
        COUNTS["backend: " + ("cuda" if gpu else "host build of the node routines")] = 1
        for name in ("Mpfa", "Mpsa", "Biot", "Tpfa", "Upwind", "Tpsa", "MVEM", "RT0"):
            for owner, tag in ((getattr(fv, name), "porepy_b200"), (getattr(pp, name), "reference")):
                stock = owner.discretize

                def counted(self, sd, data, _stock=stock, _tag=tag, _name=name):
                    out = _stock(self, sd, data)   # counted only when it returns (no NotImplementedError)
                    COUNTS[f"{_name}.discretize on the {_tag} path"] += 1
                    return out
                owner.discretize = counted
        import importlib
        hybrid = importlib.import_module(pp.__name__ + ".numerics.vem.hybrid")
        for owner, tag in ((fv.HybridDualVEM, "porepy_b200"), (hybrid.HybridDualVEM, "reference")):
            stock = owner.matrix_rhs

            def counted_matrix_rhs(self, g, data, _stock=stock, _tag=tag):
                out = _stock(self, g, data)
                COUNTS[f"HybridDualVEM.matrix_rhs on the {_tag} path"] += 1
                return out
            owner.matrix_rhs = counted_matrix_rhs
        if "--stock" in sys.argv:  # control run: the unmodified reference in the same environment
            COUNTS["classes: stock reference (control run)"] = 1
            return
        # the reference's tests also cover what porepy_b200 refuses (periodic faces, sub-face boundary
        # conditions): opt into the counted hand-over so that those tests still run, and report every reason
        self.b200 = plugin(pp, allow_reference_fallback=True)
        self.b200.install()

    def pytest_terminal_summary(self, terminalreporter):
        terminalreporter.write_line("")
        for k in sorted(COUNTS):
            terminalreporter.write_line(f"[porepy_b200] {k}: {COUNTS[k]}")
        for k, v in sorted(getattr(getattr(self, "b200", None), "fallback_calls", {}).items()):
            terminalreporter.write_line(f"[porepy_b200] handed to the reference ({v}x): {k}")


if __name__ == "__main__":
    import pytest
    if not os.path.isdir(REF_TESTS):
        sys.exit("reference tree not present")
    # extra arguments: reference test files (relative to /root/reference/tests) and pytest options
    extra = [a for a in sys.argv[1:] if a.endswith(".py") or "::" in a]
    opts = [a for a in sys.argv[1:] if a not in extra and a != "--stock"]
    if extra:
        files = [os.path.join("/root/reference/tests", a) for a in extra]
    else:
        files = [os.path.join(REF_TESTS, f) for f in ("test_mpfa.py", "test_mpsa.py", "test_biot.py", "test_tpsa.py")]
    os.chdir("/tmp")
    sys.exit(pytest.main(files + ["-p", "no:cacheprovider", "-o", "addopts=", "-q", "--rootdir", "/tmp", *opts],
                         plugins=[Rebind()]))
