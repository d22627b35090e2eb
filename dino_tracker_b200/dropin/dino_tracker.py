"""``dino_tracker`` drop-in: the reference's ``DINOTracker`` with its three best-buddy contrastive losses on libdinotrk.

With ``dino_tracker_b200/dropin`` ahead of the reference root on ``sys.path`` (INTEGRATION.md), the reference's
``train.py`` imports this module; it loads the reference's own ``dino_tracker.py`` from the rest of ``sys.path`` and
re-exports ``DINOTracker`` as a subclass that rebinds only ``get_bb_pairs_contrastive_loss``,
``get_dino_bb_contrastive_loss`` and ``get_refined_bb_contrastive_loss`` (dino_tracker_b200/contrastive.py).  Every other
attribute is the reference's object."""
import importlib.util
import os
import sys

_here = os.path.dirname(os.path.abspath(__file__))
_repo = os.path.dirname(os.path.dirname(_here))
if _repo not in sys.path:
    sys.path.append(_repo)  # so that ``import dino_tracker_b200`` resolves


def _load_reference():
    for p in sys.path:
        cand = os.path.join(os.path.abspath(p or "."), "dino_tracker.py")
        if os.path.dirname(cand) != _here and os.path.isfile(cand):
            spec = importlib.util.spec_from_file_location("_reference_dino_tracker", cand)
            mod = importlib.util.module_from_spec(spec)
            sys.modules[spec.name] = mod
            spec.loader.exec_module(mod)
            return mod
    raise ImportError("the reference's dino_tracker.py is not on sys.path after the drop-in directory")


_reference = _load_reference()

from dino_tracker_b200 import contrastive as _cl  # noqa: E402


class DINOTracker(_reference.DINOTracker):
    get_bb_pairs_contrastive_loss = _cl.get_bb_pairs_contrastive_loss
    get_dino_bb_contrastive_loss = _cl.get_dino_bb_contrastive_loss
    get_refined_bb_contrastive_loss = _cl.get_refined_bb_contrastive_loss


DINOTracker.__module__ = __name__
