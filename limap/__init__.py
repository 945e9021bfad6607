"""Import alias so that code written against the reference package (`import limap.triangulation`,
`limap.optimize`, `limap.base`, `limap.vplib`) resolves to the H100 engine's operator surface.
Only the hot-path packages exist; everything else of cvg/limap is out of scope (DESIGN.md)."""
import importlib
import sys

for _name in ("base", "triangulation", "optimize", "vplib", "merging", "util", "util.io", "runners", "visualize", "pointsfm",
              "evaluation", "estimators"):
    try:
        _m = importlib.import_module(f"limap_b200.{_name}")
    except ModuleNotFoundError:
        continue
    sys.modules[f"limap.{_name}"] = _m
    if "." not in _name:
        globals()[_name] = _m
# optimize/hybrid_localization is a subpackage of the reference's optimize package
if "limap.optimize" in sys.modules:
    sys.modules["limap.optimize.hybrid_localization"] = sys.modules["limap_b200.hybrid_localization"]
    sys.modules["limap.optimize.hybrid_localization.solve"] = sys.modules["limap_b200.hybrid_localization"]
    _fn = importlib.import_module("limap_b200.hybrid_localization_functions")
    sys.modules["limap.optimize.hybrid_localization.functions"] = _fn
    sys.modules["limap_b200.hybrid_localization"].functions = _fn
