"""CPU: the trajectory and flow-filter oracles against the live reference's vectors, bit for bit; and the flow-filter
oracle on hand-built nearest-trajectory cases (NaN trajectories, equidistant ties, an all-NaN frame)."""
import os

import numpy as np
import torch

from oracle import make_golden_preprocess as mgp
from oracle import of_filter as oof
from oracle import trajectories as otr

from golden_util import GOLDEN_DIR


def _traj_case(name):
    cfg = mgp.TRAJ_CASES[name]
    g = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    assert g["cfg"].tolist() == [cfg["H"], cfg["W"], cfg["T"], cfg["seed"], cfg["min_len"]]
    fwd, bwd, direct = otr.stack_flows(mgp.traj_case_flows(cfg), cfg["T"])
    res = otr.extract_trajectories(fwd, bwd, direct if cfg["direct"] else None, cfg["threshold"], cfg["min_len"], cfg["dthr"])
    return res, g["trajectories"]


def test_chaining_with_look_behind_matches_reference():
    res, ref = _traj_case("traj_chain_small")
    assert res.shape == ref.shape and np.array_equal(res.numpy(), ref, equal_nan=True)


def test_chaining_with_direct_flow_matches_reference():
    res, ref = _traj_case("traj_direct_small")
    assert res.shape == ref.shape and np.array_equal(res.numpy(), ref, equal_nan=True)


def test_of_filter_matches_reference():
    traj, bb = mgp.of_case_inputs()
    res = oof.of_filter(bb, traj, mgp.OF_CASE["H"], mgp.OF_CASE["W"], mgp.OF_CASE["stride"])
    ref = dict(np.load(os.path.join(GOLDEN_DIR, "of_filter_small.npz")))
    got = {f"{k}.{kk}": vv.numpy() for k, v in res.items() for kk, vv in v.items() if vv is not None}
    assert set(got) == set(ref)
    assert any(k.endswith(".r") for k in ref) and any(k.endswith(".cos_sims") for k in ref)
    for k in ref:
        assert np.array_equal(got[k], ref[k]), k


def nearest_cases():
    """Trajectories [M][T][2] built so that frame 0 has NaN trajectories in front of the nearest one, frame 1 has
    exact equidistant ties between non-adjacent indices, frame 2 is all NaN."""
    M, T = 6, 3
    traj = torch.full((M, T, 2), float("nan"))
    traj[3, 0] = torch.tensor([8.0, 8.0])
    traj[5, 0] = torch.tensor([30.0, 20.0])
    traj[1, 1] = torch.tensor([7.0, 10.0])     # (7, 7) is 3 away from both
    traj[4, 1] = torch.tensor([10.0, 7.0])
    traj[2, 1] = torch.tensor([4.0, 7.0])
    return traj


def test_nearest_oracle_on_built_cases():
    traj = nearest_cases()
    near = oof.nearest_grid(traj, 40, 40, 7)
    assert near[0, 0, 0] == 3 and near[0, 1, 3] == 5      # (7, 7) -> index 3; (28, 14) -> index 5
    assert near[1, 0, 0] == 1                            # ties at 3 px: indices 1, 2, 4 -> 1
    assert (near[2] == 0).all()                          # all NaN -> 0
