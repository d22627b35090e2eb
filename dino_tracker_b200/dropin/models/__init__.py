"""Drop-in ``models`` package: put ``dino_tracker_b200/dropin`` in front of the reference root on
``PYTHONPATH`` and the reference's ``inference_grid.py`` / ``inference_benchmark.py`` /
``dino_tracker.py`` pick up this project's ``models.tracker`` and ``models.model_inference`` unchanged
(INTEGRATION.md).  Every other ``models.*`` module (``models.utils``, ``models.networks``,
``models.extractor``) falls through to the reference tree: its ``models`` directory is appended to this
package's search path when it is importable."""
import os
import sys

_here = os.path.dirname(os.path.abspath(__file__))
_repo = os.path.dirname(os.path.dirname(os.path.dirname(_here)))
if _repo not in sys.path:
    sys.path.append(_repo)  # so that ``import dino_tracker_b200`` resolves

for _p in list(sys.path):
    _cand = os.path.join(_p or ".", "models")
    if os.path.isfile(os.path.join(_cand, "model_inference.py")) and \
            os.path.abspath(_cand) != _here and os.path.isdir(os.path.join(_cand, "networks")):
        __path__.append(os.path.abspath(_cand))
        break
