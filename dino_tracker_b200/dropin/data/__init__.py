"""Drop-in ``data`` package: with ``dino_tracker_b200/dropin`` in front of the reference root on ``PYTHONPATH``, the
reference's ``dino_tracker.py`` imports this project's ``data.dataset`` (the training-batch sampler on libdinotrk)
unchanged (INTEGRATION.md).  Every other ``data.*`` module (``data.data_utils``, ``data.tapvid``) falls through to the
reference tree: its ``data`` directory is appended to this package's search path when it is importable."""
import os
import sys

_here = os.path.dirname(os.path.abspath(__file__))
_repo = os.path.dirname(os.path.dirname(os.path.dirname(_here)))
if _repo not in sys.path:
    sys.path.append(_repo)  # so that ``import dino_tracker_b200`` resolves

for _p in list(sys.path):
    _cand = os.path.join(_p or ".", "data")
    if os.path.abspath(_cand) != _here and os.path.isfile(os.path.join(_cand, "dataset.py")) and \
            os.path.isfile(os.path.join(_cand, "data_utils.py")):
        __path__.append(os.path.abspath(_cand))
        break
