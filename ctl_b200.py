"""Import alias: ``import ctl_b200`` == the package in ``centroids-reid_b200/`` (whose
mandated directory name is not a valid Python identifier)."""
import importlib
import os
import sys

_root = os.path.dirname(os.path.abspath(__file__))
if _root not in sys.path:
    sys.path.insert(0, _root)
_pkg = importlib.import_module("centroids-reid_b200")


def _alias(name):
    """`ctl_b200.a.b` -> the SAME module object as `centroids-reid_b200.a.b`."""
    real = importlib.import_module("centroids-reid_b200" + (("." + name) if name else ""))
    sys.modules["ctl_b200" + (("." + name) if name else "")] = real
    return real


for _sub in ("_native", "retrieval", "utils", "utils.reid_metric", "utils.eval_reid", "losses",
             "losses.triplet_loss", "losses.center_loss", "reduce", "modelling", "inference", "datasets",
             "datasets.transforms"):
    try:
        _alias(_sub)
    except ModuleNotFoundError:
        pass
sys.modules["ctl_b200"] = _pkg
