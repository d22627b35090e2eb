"""Golden trace of the training loop's control flow -> tests/golden/train_loop_trace.npz.

Runs the live reference's ``DINOTracker.train()`` (dino_tracker.py:392-448) through ``oracle/ref_harness.py`` on the CPU
with cheap stand-ins for the model, the sampler and every loss term (tiny tensors with gradients into two small
parameter groups, so Adam and the ``LambdaLR`` schedule run for real), and records per iteration: i, the terms called in
order, both parameter groups' lr after the scheduler step; and per run: the start iteration, the scheduler steps before
the loop, the checkpoints loaded and written, the ``load_next_batch`` calls and the log steps.

``native_trace`` runs ``dino_tracker_b200.trainer.DinoTrackerTrainer.train()`` with the same stand-ins and records the
same trace (tests/test_trainer_loop_cpu.py); it needs neither the reference nor a GPU.

    python oracle/make_golden_train_loop.py [--out tests/golden/train_loop_trace.npz]
"""
import argparse
import contextlib
import os
import sys
import tempfile

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# small thresholds, so that a few iterations cross every rule of the loop
CONFIG = {"video_resw": 8, "video_resh": 6, "keep_traj_in_cpu": False, "fg_traj_ratio": 0.5, "train_batch_size": 4,
          "batch_n_frames": 2, "checkpoint_interval": 3, "sampler_batch_iterations": 2, "lr_delta_dino": 0.01,
          "lr_cnn_refiner": 0.02, "apply_scheduler_every": 2, "scheduler_gamma": 0.9, "lambda_cyc": 0.5, "apply_cyc_after": 2,
          "cyc_n_frames": 2, "cyc_batch_size_per_frame": 4, "cyc_fg_points_ratio": 0.5, "cyc_thresh": 4, "cyc_gamma": 0.8,
          "lambda_emb_norm": 0.0001, "lambda_angle": 0.0001, "lambda_cl_dino_bb": 0.00025, "lambda_cl_ref_bb": 0.00005,
          "cl_n_frames": 2, "cl_points_per_pair": 4, "cl_fg_points_ratio": 0.5, "cl_temp": 0.1, "cl_div_dino_bb": 700,
          "cl_div_ref_bb": 900, "apply_cl_ref_after": 4, "bb_amb_sig_a": 27, "bb_amb_sig_b": -5.7, "stride": 7,
          "dino_patch_size": 14}
# (total_iterations, checkpoint already in the folder or None)
CASES = {"fresh_7": (7, None), "ckpt0_7": (7, 0), "ckpt3_7": (7, 3), "fresh_205": (205, None)}


class Recorder:
    def __init__(self):
        self.i = None
        self.iters, self.terms, self.lr = [], [], []
        self.pre_loop_steps, self.loaded, self.saved, self.next_batch, self.logs = 0, [], [], [], []

    def loop(self, it):
        """stands in for ``tqdm`` around the loop's range"""
        for i in it:
            self.i = i
            self.iters.append(i)
            self.terms.append([])
            self.lr.append([np.nan, np.nan])
            yield i

    def call(self, name):
        self.terms[-1].append(name)

    def scheduler(self, make):
        def wrapped(optimizer, **kw):
            s = make(optimizer, **kw)
            step = s.step

            def recorded_step():
                step()
                if self.i is None:
                    self.pre_loop_steps += 1
                else:
                    self.lr[-1] = [g["lr"] for g in optimizer.param_groups]
            s.step = recorded_step
            return s
        return wrapped

    def arrays(self, prefix):
        return {prefix + "iters": np.array(self.iters, np.int64),
                prefix + "terms": np.array([" ".join(t) for t in self.terms]),
                prefix + "lr": np.array(self.lr, np.float64).reshape(-1, 2),
                prefix + "pre_loop_steps": np.array(self.pre_loop_steps, np.int64),
                prefix + "loaded": np.array(self.loaded, np.int64), prefix + "saved": np.array(self.saved, np.int64),
                prefix + "next_batch": np.array(self.next_batch, np.int64), prefix + "logs": np.array(self.logs, np.int64)}


class StandInModel(nn.Module):
    """Two parameter groups named as the tracker's; ``forward`` maps the source points' (x, y) through both."""

    def __init__(self, rec, **_):
        super().__init__()
        self.rec = rec
        self.delta_dino = nn.Linear(2, 2)
        self.tracker_head = nn.Linear(2, 2)
        with torch.no_grad():
            for p, v in ((self.delta_dino.weight, [[0.5, -0.2], [0.1, 0.3]]), (self.delta_dino.bias, [0.01, -0.02]),
                         (self.tracker_head.weight, [[0.2, 0.1], [-0.4, 0.6]]), (self.tracker_head.bias, [0.03, 0.0])):
                p.copy_(torch.tensor(v))

    def forward(self, inputs):
        self.rec.call("track")
        return self.tracker_head(self.delta_dino(inputs[0][:, :2]))

    def save_weights(self, k):
        self.rec.saved.append(k)

    def load_weights(self, k):
        self.rec.loaded.append(k)


class StandInSampler:
    def __init__(self, rec, **_):
        self.rec = rec

    def __call__(self):
        self.rec.call("sample")
        g = torch.Generator().manual_seed(len(self.rec.iters))
        t1 = torch.rand(4, 3, generator=g)
        return {"t1_points": t1, "t2_points_normalized": torch.rand(4, 3, generator=g) * 2 - 1,
                "source_frame_indices": torch.tensor([0, 1, 0, 1]), "target_frame_indices": torch.tensor([1, 0, 1, 0]),
                "frames_set_t": torch.tensor([0, 1], dtype=torch.int32)}

    def load_next_batch(self):
        self.rec.next_batch.append(self.rec.i)


def _term(rec, name, fn):
    def term(model, *a, **kw):
        rec.call(name)
        return fn(model)
    return term


def _cyc(m):
    return (m.delta_dino.weight ** 2).sum() * 0.5


def _ref(m):
    return m.tracker_head.weight.abs().sum() * 0.1


def _dino(m):
    return (m.delta_dino.bias ** 2).sum() + m.tracker_head.bias.sum()


def _norm(m):
    return m.delta_dino.weight.sum() ** 2 * 0.01


def _angle(m):
    return (m.tracker_head.bias ** 2).sum()


def make_folder(root, ckpt):
    """A data folder with one 8 x 6 frame (the trainers read the frame count) and, optionally, checkpoint ``ckpt``."""
    from PIL import Image
    os.makedirs(os.path.join(root, "video"), exist_ok=True)
    Image.fromarray(np.zeros((6, 8, 3), np.uint8)).save(os.path.join(root, "video", "00000.png"))
    folder = os.path.join(root, "models", "dino_tracker")
    os.makedirs(folder, exist_ok=True)
    if ckpt is not None:
        for name in (f"tracker_head_{ckpt}.pt", f"delta_dino_{ckpt}.pt"):
            open(os.path.join(folder, name), "wb").close()
    return root


@contextlib.contextmanager
def _patched(module, **attrs):
    old = {k: getattr(module, k) for k in attrs}
    for k, v in attrs.items():
        setattr(module, k, v)
    try:
        yield
    finally:
        for k, v in old.items():
            setattr(module, k, v)


def _config(total):
    return dict(CONFIG, total_iterations=total)


def native_trace(case, workdir):
    """The trace of ``DinoTrackerTrainer.train()`` (on the CPU) with the stand-ins, for CASES[case] in ``workdir``."""
    from dino_tracker_b200 import trainer as tm
    total, ckpt = CASES[case]
    rec = Recorder()
    tr = tm.DinoTrackerTrainer(_config(total), make_folder(workdir, ckpt), device="cpu")
    tr.load_fg_masks = lambda: None
    tr.load_dino_best_buddies = lambda: None
    tr.get_sampler = lambda: StandInSampler(rec)
    tr.get_model = lambda: StandInModel(rec)
    tr.cycle_loss = _term(rec, "cyc", _cyc)
    tr.refined_bb_loss = _term(rec, "ref", _ref)
    tr.dino_bb_loss = _term(rec, "dino", _dino)
    tr.regularisers = _term(rec, "reg", lambda m: (_norm(m), _angle(m)))
    log = tr.log_losses
    tr.log_losses = lambda i: (rec.logs.append(i), log(i))
    with _patched(tm, tqdm=rec.loop, get_cnn_refiner_scheduler=rec.scheduler(tm.get_cnn_refiner_scheduler)):
        tr.train()
    return rec.arrays("")


def reference_trace(case, workdir):
    """The same trace of the live reference's ``DINOTracker.train()``."""
    import yaml
    sys.path.insert(0, ROOT)
    from oracle import ref_harness
    ref_harness.install("cpu")
    import dino_tracker as dt
    total, ckpt = CASES[case]
    rec = Recorder()
    cfg_path = os.path.join(workdir, "train.yaml")
    with open(cfg_path, "w") as f:
        yaml.safe_dump(_config(total), f)
    args = argparse.Namespace(config=cfg_path, data_path=make_folder(workdir, ckpt))
    with _patched(dt, tqdm=rec.loop, get_cnn_refiner_scheduler=rec.scheduler(dt.get_cnn_refiner_scheduler),
                  Tracker=lambda **kw: StandInModel(rec), load_video=lambda *a, **kw: torch.zeros(1, 3, 6, 8),
                  DinoTrackerSampler=lambda **kw: StandInSampler(rec)):
        tr = dt.DINOTracker(args)
        tr.load_fg_masks = lambda: None
        tr.load_dino_best_buddies = lambda: None
        tr.load_trajectories = lambda: (None, None)
        tr.get_cycle_consistency_loss = _term(rec, "cyc", _cyc)
        tr.get_refiner_contrastive_loss = _term(rec, "ref", _ref)
        tr.get_dino_bb_contrastive_loss = _term(rec, "dino", _dino)
        tr.get_emb_norm_regularization_loss = _term(rec, "reg", _norm)   # the two reference terms are one call natively
        tr.get_emb_angle_regularization_loss = lambda m: _angle(m)
        log = tr.log_losses
        tr.log_losses = lambda i, log_interval=100: (rec.logs.append(i), log(i, log_interval=log_interval))
        tr.train()
    return rec.arrays("")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "train_loop_trace.npz"))
    args = ap.parse_args()
    out = {}
    for case in CASES:
        with tempfile.TemporaryDirectory() as d:
            out.update({f"{case}/{k}": v for k, v in reference_trace(case, d).items()})
    np.savez_compressed(args.out, **out)
    print(f"wrote {args.out}: {', '.join(f'{c} ({len(out[c + '/iters'])} iterations)' for c in CASES)}")


if __name__ == "__main__":
    main()
