"""``models.tracker`` drop-in: the CUDA Tracker under the reference's module path."""
from dino_tracker_b200.tracker import EPS, Tracker  # noqa: F401
