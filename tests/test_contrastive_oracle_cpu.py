"""CPU suite: the oracle of the best-buddy contrastive losses (oracle/contrastive.py) reproduces the live reference's
fixture (tests/golden/contrastive_small.npz) in loss, gradient and selected indices; where the reference tree is present
the fixture regenerates bit for bit and the drop-in ``dino_tracker`` rebinds exactly the three loss methods."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import contrastive as oc
from oracle import make_golden_contrastive as mg
from oracle import ref_harness

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "contrastive_small.npz")

OracleTrainer = type("OracleTrainer", (), {n: getattr(oc, n) for n in (
    "get_dino_bb_contrastive_loss", "get_refined_bb_contrastive_loss", "get_bb_pairs_contrastive_loss")})


@pytest.mark.parametrize("which", ["dino", "refined"])
def test_oracle_reproduces_fixture(which):
    z = np.load(GOLDEN)
    emb = torch.from_numpy(z["emb"])
    tr = mg.trainer_standin(OracleTrainer, torch.from_numpy(z["masks"]), mg.load_bb(z))
    video = torch.zeros(mg.T, 3, *z["video_hw"].tolist())
    rec = []
    loss, grad = mg.run_loss(which, OracleTrainer, tr, emb, video, int(z[f"{which}_seed"]), rec)
    pairs, src, tgt = mg.pack_record(rec)
    assert np.array_equal(pairs, z[f"{which}_pairs"])
    assert np.array_equal(src, z[f"{which}_src"]) and np.array_equal(tgt, z[f"{which}_tgt"])
    torch.testing.assert_close(loss, torch.from_numpy(z[f"{which}_loss"]), rtol=1e-5, atol=0)
    torch.testing.assert_close(grad, torch.from_numpy(z[f"{which}_grad"]), rtol=1e-4, atol=1e-8)


def test_fixture_cases():
    z = np.load(GOLDEN)
    frames = z["frames"]
    assert any(s == t for s, t, _ in z["refined_pairs"]), "no refined self-pair"
    assert any(frames[s] == mg.EMPTY_MASK_FRAME for s, _, _ in z["dino_pairs"]), "no dino-BB pair without fg buddies"


@pytest.mark.skipif(not ref_harness.reference_available(), reason="reference tree not present")
def test_fixture_regenerates_bit_for_bit():
    z = np.load(GOLDEN)
    new = mg.generate()
    assert set(new) == set(z.files)
    for k in z.files:
        assert np.array_equal(np.asarray(new[k]), z[k]), k


@pytest.mark.skipif(not ref_harness.reference_available(), reason="reference tree not present")
def test_dropin_rebinds_exactly_the_three_losses():
    code = f"""
import sys
sys.path[:0] = [{os.path.join(ROOT, 'dino_tracker_b200', 'dropin')!r}, {ref_harness.REFERENCE_ROOT!r}]
from oracle import ref_harness
for name in ("imageio", "imageio.v3", "matplotlib", "matplotlib.pyplot", "antialiased_cnns"):
    import types; m = types.ModuleType(name); m.BlurPool = object; sys.modules.setdefault(name, m)
import dino_tracker as d
from dino_tracker_b200 import contrastive as c
ref = sys.modules["_reference_dino_tracker"].DINOTracker
assert issubclass(d.DINOTracker, ref) and d.DINOTracker.__mro__[1] is ref
own = {{k for k in vars(d.DINOTracker) if not k.startswith("__")}}
assert own == {{"get_bb_pairs_contrastive_loss", "get_dino_bb_contrastive_loss", "get_refined_bb_contrastive_loss"}}, own
for k in own:
    assert getattr(d.DINOTracker, k) is getattr(c, k)
for k in vars(ref):
    if k not in own and not k.startswith("__"):
        assert getattr(d.DINOTracker, k) is getattr(ref, k), k
print("ok")
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr
