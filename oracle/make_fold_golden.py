"""Generate tests/golden/fold_ref.json by RUNNING the reference's north-fold helpers (xgcm/padding.py:21-181).

    XGCM_REFERENCE_ROOT=<xgcm checkout> python -m oracle.make_fold_golden

Records ``_seam_partner_indices`` for every seam position x pivot seam role x a few lengths,
``_resolve_pivot`` for every alias and a few explicit mappings, and whether ``_parse_fold_padding`` accepts
(with its normalised result) or raises on good and bad specs.  The helpers are pure numpy; ``xgcm.padding``
only needs xarray for def-time annotations, so it is imported with the stand-in module of
``oracle/ref_loader.py`` without running ``xgcm/__init__.py``.  Nothing is copied.

TEST INFRASTRUCTURE ONLY.
"""

from __future__ import annotations

import importlib
import json
import sys
import types
from pathlib import Path

from . import ref_loader

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden" / "fold_ref.json"

# (label, spec): a raising spec records the exception type and message
FOLD_SPECS = [
    ("corner", {"fold": "corner"}),
    ("T_south_periodic", {"fold": "T", "south": "periodic"}),
    ("u_south_extend", {"fold": "u", "south": "extend"}),
    ("explicit", {"fold": {"X": "right", "Y": "center"}}),
    ("explicit_outer", {"fold": {"X": "outer", "Y": "inner"}, "south": "fill"}),
    ("unknown_alias", {"fold": "banana"}),
    ("british_centre", {"fold": {"X": "centre", "Y": "center"}}),
    ("bad_position", {"fold": {"X": "banana"}}),
    ("empty_mapping", {"fold": {}}),
    ("bad_south", {"fold": "corner", "south": "wrap"}),
    ("extra_key", {"fold": "corner", "north": "fill"}),
    ("not_a_pivot", {"fold": 3}),
    ("no_fold_key", {"south": "fill"}),
]


def load_padding():
    """The reference's ``xgcm.padding`` module, imported as it lies on disk."""
    if not ref_loader.available():
        raise RuntimeError("set XGCM_REFERENCE_ROOT to a checkout of the xgcm source tree")
    added = []
    if "xarray" not in sys.modules:
        sys.modules["xarray"] = ref_loader._stub(
            "xarray", DataArray=type("DataArray", (), {}), Dataset=type("Dataset", (), {})
        )
        added.append("xarray")
    pkg = types.ModuleType("xgcm")
    pkg.__path__ = [str(ref_loader.REFERENCE_ROOT / "xgcm")]
    prev = sys.modules.get("xgcm")
    sys.modules["xgcm"] = pkg
    try:
        return importlib.import_module("xgcm.padding")
    finally:
        for name in list(sys.modules):
            if name == "xgcm" or name.startswith("xgcm."):
                del sys.modules[name]
        if prev is not None:
            sys.modules["xgcm"] = prev
        for name in added:
            sys.modules.pop(name, None)


def fold_reference(padding):
    partners = {}
    for position in ("center", "left", "right", "outer", "inner"):
        for role in ("center", "edge"):
            for length in (2, 3, 5, 8, 9):
                idx = padding._seam_partner_indices(position, role, length)
                partners[f"{position}|{role}|{length}"] = [int(v) for v in idx]
    pivots = {}
    for alias in ("center", "T", "t", "corner", "F", "f", "U", "u", "V", "v", "Center", "CORNER"):
        pivots[alias] = padding._resolve_pivot(alias, "Y", "X")
    explicit = [{"X": "right", "Y": "center"}, {"X": "left", "Y": "left"}, {"X": "right", "Y": "right"},
                {"X": "outer"}, {"Y": "inner"}, {"X": "center", "Y": "outer"}]
    for m in explicit:
        pivots[json.dumps(m, sort_keys=True)] = padding._resolve_pivot(m, "Y", "X")
    specs = {}
    for label, spec in FOLD_SPECS:
        try:
            specs[label] = {"spec": spec, "result": padding._parse_fold_padding(spec)}
        except Exception as err:  # the outcome is the datum
            specs[label] = {"spec": spec, "raises": type(err).__name__, "message": str(err)}
    return {"partners": partners, "pivots": pivots, "specs": specs}


def main():
    GOLDEN.write_text(json.dumps(fold_reference(load_padding()), indent=1, sort_keys=True))
    print(GOLDEN.name, GOLDEN.stat().st_size)


if __name__ == "__main__":
    main()
