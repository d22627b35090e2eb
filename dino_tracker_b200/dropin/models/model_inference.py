"""``models.model_inference`` drop-in: the CUDA inference driver under the reference's module path."""
from dino_tracker_b200.model_inference import (ModelInference, generate_trajectories,  # noqa: F401
                                               generate_trajectory, generate_trajectory_input)
