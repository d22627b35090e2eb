"""``data.dataset`` drop-in: ``DinoTrackerSampler`` is the library's (dino_tracker_b200/sampler.py); ``RangeNormalizer``
and ``LongRangeSampler`` are the reference's own objects, from its ``data/dataset.py`` loaded under a private module
name from the rest of ``sys.path``."""
import importlib.util
import os
import sys

_here = os.path.dirname(os.path.abspath(__file__))


def _load_reference():
    for p in sys.path:
        cand = os.path.join(os.path.abspath(p or "."), "data", "dataset.py")
        if os.path.dirname(cand) != _here and os.path.isfile(cand):
            spec = importlib.util.spec_from_file_location("_reference_data_dataset", cand)
            mod = importlib.util.module_from_spec(spec)
            sys.modules[spec.name] = mod
            spec.loader.exec_module(mod)
            return mod
    raise ImportError("the reference's data/dataset.py is not on sys.path after the drop-in directory")


_reference = _load_reference()
RangeNormalizer = _reference.RangeNormalizer
LongRangeSampler = _reference.LongRangeSampler

from dino_tracker_b200.sampler import DinoTrackerSampler  # noqa: E402,F401
