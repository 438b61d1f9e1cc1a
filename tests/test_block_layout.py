"""``porepy_b200.layout.BlockLayout`` on a small hand-built layout: part offsets, slicing by name, entry numbers of cells,
the parts listed for the model bridges, and the refusals of ``stack``."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from porepy_b200.layout import BlockLayout

M, F0, F1, I0 = ("matrix",), ("fracture", 0), ("fracture", 1), ("interface", 0)


def _layout():
    return BlockLayout([("pressure", [(M, 4, 1), (F0, 2, 1), (F1, 1, 1)]), ("displacement", [(M, 4, 3)]),
                        ("interface_displacement", [(I0, 3, 2)])])


def test_offsets_parts_and_items():
    lay = _layout()
    assert lay.size == 4 + 2 + 1 + 12 + 6
    assert lay.offsets.tolist() == [0, 4, 6, 7, 19, 25]
    x = np.arange(lay.size) * 10
    parts = lay.parts(x)
    assert list(parts) == ["pressure", "displacement", "interface_displacement"]
    assert [p.tolist() for p in parts["pressure"]] == [[0, 10, 20, 30], [40, 50], [60]]
    assert parts["displacement"][0].tolist() == list(range(70, 190, 10))
    assert np.shares_memory(parts["interface_displacement"][0], x)              # views, as a slice gives
    assert lay.items() == [("pressure", M, 4, 1), ("pressure", F0, 2, 1), ("pressure", F1, 1, 1),
                           ("displacement", M, 4, 3), ("interface_displacement", I0, 3, 2)]


def test_span():
    lay = _layout()
    assert lay.span("pressure", F0, [1, 0]).tolist() == [[5], [4]]
    assert lay.span("displacement", M, [0, 2]).tolist() == [[7, 8, 9], [13, 14, 15]]
    assert lay.span("interface_displacement", I0, np.array([2])).tolist() == [[23, 24]]
    assert lay.span("pressure", M, []).shape == (0, 1)


def test_insert():
    lay = _layout().insert("pressure", [("temperature", [(M, 4, 1)])])
    assert [name for name, _ in lay.blocks] == ["pressure", "temperature", "displacement", "interface_displacement"]
    assert lay.span("displacement", M, [0]).tolist() == [[11, 12, 13]]


def _values(*sizes):
    return [SimpleNamespace(val=torch.zeros(n)) for n in sizes]


def test_stack_orders_and_checks_lengths():
    lay = _layout()
    p, u, uj = _values(4, 2, 1), _values(12), _values(6)
    out = lay.stack({"interface_displacement": uj, "displacement": u, "pressure": p})
    assert [id(v) for v in out] == [id(v) for v in p + u + uj]
    with pytest.raises(ValueError, match="interface_displacement: None entries per part"):
        lay.stack({"pressure": p, "displacement": u})                                   # a missing block
    with pytest.raises(ValueError, match="temperature"):
        lay.stack({"pressure": p, "displacement": u, "interface_displacement": uj, "temperature": p})
    with pytest.raises(ValueError, match=r"pressure: \[4, 2\] entries per part, the layout has \[4, 2, 1\]"):
        lay.stack({"pressure": p[:2], "displacement": u, "interface_displacement": uj})
    with pytest.raises(ValueError, match=r"pressure: \[4, 2, 2\]"):
        lay.stack({"pressure": _values(4, 2, 2), "displacement": u, "interface_displacement": uj})   # wrong length
