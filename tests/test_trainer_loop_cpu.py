"""CPU suite: the native training loop's control flow (dino_tracker_b200/trainer.py) against a committed trace of the live
reference's ``DINOTracker.train()`` (oracle/make_golden_train_loop.py), with the same stand-ins for the model, the
sampler and the loss terms: the iterations run, the terms called in order, both lr groups after every scheduler step, the
checkpoints loaded and written, the ``load_next_batch`` calls and the log steps must all be identical, for a fresh
folder, a folder holding checkpoint 0 and one holding checkpoint 3."""
import os

import numpy as np
import pytest

from oracle import make_golden_train_loop as mg
from oracle import ref_harness

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_loop_trace.npz")


def _golden(case):
    g = np.load(GOLDEN)
    return {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(case + "/")}


def _assert_same(got, want):
    assert set(got) == set(want)
    for k in want:
        assert got[k].dtype.kind == want[k].dtype.kind and np.array_equal(got[k], want[k]), \
            f"{k}: {got[k].tolist()} != {want[k].tolist()}"


@pytest.mark.parametrize("case", list(mg.CASES))
def test_native_loop_matches_reference_trace(case, tmp_path):
    _assert_same(mg.native_trace(case, str(tmp_path)), _golden(case))


def test_checkpoint_discovery_reads_only_checkpoints(tmp_path):
    from dino_tracker_b200.trainer import last_ckpt_iter
    assert last_ckpt_iter(str(tmp_path)) == -1
    for name in ("tracker_head_40.pt", "delta_dino_40.pt", "delta_dino_7.pt", "notes.txt", "tracker_head_9.pt.tmp"):
        (tmp_path / name).write_bytes(b"")
    assert last_ckpt_iter(str(tmp_path)) == 40


@pytest.mark.skipif(not ref_harness.reference_available(), reason="needs the reference tree")
@pytest.mark.parametrize("case", list(mg.CASES))
def test_reference_reproduces_golden(case, tmp_path):
    _assert_same(mg.reference_trace(case, str(tmp_path)), _golden(case))
