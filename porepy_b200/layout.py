"""Named blocks of consecutive entries: the order and size of a model's unknowns or equations, stated once."""
from __future__ import annotations

import numpy as np


class BlockLayout:
    """``BlockLayout([(name, [(domain, count, width), ...]), ...])``: blocks (``pressure``, ``mass_balance_equation``, ...)
    in the order given, each with one part per domain, a key such as ``("matrix",)``, ``("fracture", j)``,
    ``("interface", j)`` or ``("subdomain", i)``; a part is ``count`` cells of ``width`` entries each."""

    def __init__(self, blocks):
        self.blocks = [(name, [(tuple(d), int(n), int(w)) for d, n, w in parts]) for name, parts in blocks]
        self._ends = np.concatenate(([0], np.cumsum([n * w for _, _, n, w in self.items()]))).astype(np.int64)
        self._start = {(name, d): (int(self._ends[q]), w) for q, (name, d, _, w) in enumerate(self.items())}
        self.size = int(self._ends[-1])

    @property
    def offsets(self) -> np.ndarray:
        """The part boundaries, flat, in order (one more than there are parts)."""
        return self._ends

    def items(self) -> list:
        """(name, domain, count, width) of every part, in order."""
        return [(name, d, n, w) for name, parts in self.blocks for d, n, w in parts]

    def insert(self, after: str, blocks) -> BlockLayout:
        """A new layout with ``blocks`` right behind the block ``after``."""
        i = [name for name, _ in self.blocks].index(after) + 1
        return BlockLayout(self.blocks[:i] + list(blocks) + self.blocks[i:])

    def _by_name(self, flat) -> dict:
        it = iter(flat)
        return {name: [next(it) for _ in parts] for name, parts in self.blocks}

    def parts(self, x) -> dict:
        """{name: [slice of ``x`` per part]}: views of ``x``."""
        return self._by_name([x[a:b] for a, b in zip(self._ends[:-1], self._ends[1:])])

    def variables(self, x) -> dict:
        """{name: [``DeviceAdArray`` per part]}: one ``ad.variables`` over all parts of ``x``, in order."""
        from . import ad
        return self._by_name(ad.variables([p for parts in self.parts(x).values() for p in parts]))

    def stack(self, blocks: dict) -> list:
        """{name: [value per part]} -> the values in layout order.  A missing or unknown block, or a block whose parts'
        ``val`` do not hold count x width entries each, raises ``ValueError`` (reads ``numel`` only)."""
        got = {name: [v.val.numel() for v in values] for name, values in blocks.items()}
        want = {name: [n * w for _, n, w in parts] for name, parts in self.blocks}
        bad = [f"{k}: {got.get(k)} entries per part, the layout has {want.get(k)}"
               for k in sorted(got.keys() | want.keys()) if got.get(k) != want.get(k)]
        if bad:
            raise ValueError("; ".join(bad))
        return [v for name, _ in self.blocks for v in blocks[name]]

    def span(self, name: str, domain, index) -> np.ndarray:
        """(len(index), width): the entry numbers of the cells ``index`` of the part of ``name`` on ``domain``."""
        start, w = self._start[(name, tuple(domain))]
        return start + w * np.asarray(index, np.int64)[:, None] + np.arange(w)


class LayoutModel:
    """Base of the model classes that state their unknowns in ``self.unknown_layout``."""

    @property
    def num_dofs(self) -> int:
        return self.unknown_layout.size

    @property
    def offsets(self) -> np.ndarray:
        """Boundaries of the unknowns' parts in the global vector (``unknown_layout.offsets``)."""
        return self.unknown_layout.offsets
