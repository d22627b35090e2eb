"""CPU suite: the oracle of the training-batch sampler (oracle/sampler.py) reproduces the live reference's fixture
(tests/golden/sampler_small.npz) bit for bit in both modes; where the reference tree is present the fixture regenerates
bit for bit and the drop-in ``data`` package resolves to the library's sampler and the reference's other objects."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import make_golden_sampler as mg
from oracle import ref_harness
from oracle import sampler as osm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "sampler_small.npz")


@pytest.mark.parametrize("case", sorted(mg.CASES))
def test_oracle_reproduces_fixture(case):
    z = np.load(GOLDEN)
    out, s = mg.run_case(case, osm.DinoTrackerSampler, osm.RangeNormalizer)
    assert set(out) == {k for k in z.files if k.startswith(case + "/") and not k.endswith("frame_draws")}
    for k, v in out.items():
        assert v.dtype == z[k].dtype and v.shape == z[k].shape and np.array_equal(v, z[k]), k
    assert np.array_equal(np.array(s.frame_draws), z[f"{case}/frame_draws"])


def test_fixture_cases():
    z = np.load(GOLDEN)
    c = mg.CASES["small"]
    assert z["small/frame_draws"].max() > 1, "no frame draw was redrawn"
    fg, bg = mg.case_inputs("small")
    for traj in (fg, bg):
        valid_steps = (~traj.isnan().any(-1)).sum(1)
        assert (valid_steps == 1).any(), "no single-step trajectory"
        assert (traj[..., 0].isnan() != traj[..., 1].isnan()).any(), "no NaN in one coordinate only"
    n_bg = int(((~bg.isnan().any(-1)).sum(1) > 1).sum())
    assert n_bg < c["batch"] - int(c["batch"] * c["ratio"]), "the bg set is not smaller than its share"
    n_fg = int(((~fg.isnan().any(-1)).sum(1) > 1).sum())
    assert n_fg > 0 and z["small/0/t1_points"].shape[0] < c["batch"]
    fgw, bgw = (mg.make_trajectories(n, mg.CASES["windowed"]["T"], seed, None) for n, seed, _ in
                (mg.CASES["windowed"]["fg"], mg.CASES["windowed"]["bg"]))
    for traj in (fgw, bgw):
        assert int(((~traj.isnan().any(-1)).sum(1) > 1).sum()) > osm.MAX_TRAJ_SIZE
    assert mg.CASES["windowed"]["ops"].count("next") >= 2


@pytest.mark.skipif(not ref_harness.reference_available(), reason="reference tree not present")
def test_fixture_regenerates_bit_for_bit():
    z = np.load(GOLDEN)
    new = mg.generate()
    assert set(new) == set(z.files)
    for k in z.files:
        assert new[k].dtype == z[k].dtype and np.array_equal(new[k], z[k]), k


@pytest.mark.skipif(not ref_harness.reference_available(), reason="reference tree not present")
def test_dropin_data_package():
    code = f"""
import sys
sys.path[:0] = [{os.path.join(ROOT, 'dino_tracker_b200', 'dropin')!r}, {ref_harness.REFERENCE_ROOT!r}]
import types
for name in ("imageio", "imageio.v3", "matplotlib", "matplotlib.pyplot", "antialiased_cnns"):
    m = types.ModuleType(name); m.BlurPool = object; sys.modules.setdefault(name, m)
import data.dataset as dd
import data.data_utils as du
from dino_tracker_b200 import sampler, contrastive as c
ref = sys.modules["_reference_data_dataset"]
assert dd.DinoTrackerSampler is sampler.DinoTrackerSampler
assert dd.RangeNormalizer is ref.RangeNormalizer and dd.LongRangeSampler is ref.LongRangeSampler
assert du.__file__.startswith({ref_harness.REFERENCE_ROOT!r}), du.__file__
import dino_tracker as d
assert d._reference.DinoTrackerSampler is sampler.DinoTrackerSampler
refdt = sys.modules["_reference_dino_tracker"].DINOTracker
assert d.DINOTracker.__mro__[1] is refdt
own = {{k for k in vars(d.DINOTracker) if not k.startswith("__")}}
assert own == {{"get_bb_pairs_contrastive_loss", "get_dino_bb_contrastive_loss", "get_refined_bb_contrastive_loss"}}, own
for k in own:
    assert getattr(d.DINOTracker, k) is getattr(c, k)
print("ok")
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr
