"""The training loop of DINO-Tracker on the library: ``dino_tracker.py`` (``DINOTracker``) and ``train.py`` restated.

``DinoTrackerTrainer(config, data_path, device).train()`` trains one video from the reference's on-disk layout
(``utils.add_config_paths``) and writes checkpoints the reference's and this package's ``Tracker.load_weights`` load::

    python -m dino_tracker_b200.trainer --config config/train.yaml --data-path dataset/libby --seed 2

The loop is ``dino_tracker.py:405-448`` in the reference's order, so a seeded run makes the reference's random draws:
sampler, ``model(inputs)`` and the Huber loss, the cycle term (from ``apply_cyc_after``), the refined-BB loss (from
``apply_cl_ref_after``), the dino-BB loss, the two embedding regularisers (one CUDA node, ``train.RegularisersFunction``),
backward, the Adam step and the ``LambdaLR`` step.  Checkpoint and resume rules are the reference's:

* a folder without checkpoints starts at iteration -1 and runs ``total_iterations + 1`` iterations;
* a folder whose last checkpoint is 0 loads nothing and starts at 0;
* a folder whose last checkpoint is k > 0 loads k, steps the scheduler k times and starts at k (iteration k runs again);
  Adam's moments start fresh, and the random state is not restored;
* a checkpoint is written when ``i == total_iterations - 1 or i % checkpoint_interval == 0``, and once more at
  ``total_iterations``; ``load_next_batch`` runs when ``i % sampler_batch_iterations == 0 and i > 0``.

Checkpoint discovery reads only ``tracker_head_<k>.pt`` / ``delta_dino_<k>.pt`` in ``models/dino_tracker``; the
reference's ``get_last_ckpt_iter`` fails on any other file there.  Two departures change no trained weight: the running
loss sums stay on the device and are read at each log step (``i % 100 == 0``; the reference reads seven scalars back
every iteration), and there is no per-iteration ``torch.cuda.empty_cache()``.

The loss terms (``tracking_loss``, ``cycle_loss``, ``refined_bb_loss``, ``dino_bb_loss``, ``regularisers``) and
``get_model`` / ``get_sampler`` are methods, so a test can substitute any of them.  The trainer carries ``config``,
``fg_masks`` and ``dino_bb_pairs``, which is what the ``contrastive.get_*`` losses read from it.
"""
import argparse
import logging
import os
import re
from pathlib import Path

import numpy as np
import torch
import yaml
from tqdm import tqdm

from .range_normalizer import RangeNormalizer

_CKPT = re.compile(r"(?:tracker_head|delta_dino)_(\d+)\.pt")


def fix_random_seeds(seed=31):
    """models/utils.py:98-104."""
    torch.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)
    np.random.seed(seed)


def last_ckpt_iter(folder):
    """The largest k of the ``tracker_head_<k>.pt`` / ``delta_dino_<k>.pt`` files in ``folder``, or -1 if there are none
    (models/utils.py:61-68 for a folder that holds only checkpoints)."""
    its = [int(m.group(1)) for m in (_CKPT.fullmatch(f) for f in os.listdir(folder)) if m]
    return max([-1] + its)


def get_cnn_refiner_scheduler(optimizer, gamma=0.999, apply_every=40):
    """optimization/schedulers.py: delta-DINO's lr decays by ``gamma`` every ``apply_every`` steps, the refiner's stays."""
    return torch.optim.lr_scheduler.LambdaLR(optimizer, lr_lambda=[lambda epoch: gamma ** (epoch // apply_every),
                                                                   lambda epoch: 1])


def load_video(video_folder, resize):
    """data/data_utils.py:79-104: the sorted *.jpg then *.png frames, each resized with PIL LANCZOS to ``resize`` =
    (H, W) and scaled to [0, 1] -> T x 3 x H x W fp32 (on the host)."""
    from PIL import Image
    files = sorted(list(Path(video_folder).glob("*.jpg")) + list(Path(video_folder).glob("*.png")))
    resh, resw = resize
    frames = []
    for f in files:
        img = np.array(Image.open(str(f)).resize((resw, resh), Image.LANCZOS))
        frames.append(torch.from_numpy(img).permute(2, 0, 1).float().div(255))   # transforms.ToTensor
    return torch.stack(frames)


class DinoTrackerTrainer:
    """``DINOTracker`` of dino_tracker.py on the library.  ``config``: the dict of train.yaml; ``data_path``: a folder in
    the layout ``pipeline.preprocess_video`` writes."""

    LOG_INTERVAL = 100
    _TERMS = ("loss_total", "loss_of", "loss_cl_dino_bb", "loss_cl_refiner", "loss_emb_norm_reg", "loss_angle_reg", "loss_cyc")

    def __init__(self, config, data_path, device="cuda:0"):
        self.config = config
        self.device = device
        self.set_paths(data_path)
        frames = sorted(list(Path(self.video_path).glob("*.jpg")) + list(Path(self.video_path).glob("*.png")))
        self.range_normalizer = RangeNormalizer(shapes=(config["video_resw"], config["video_resh"], len(frames)),
                                                device=device)
        self.of_loss_fn = torch.nn.HuberLoss(delta=1 / 32, reduction="none")
        self.fg_masks = None
        self.dino_bb_pairs = None
        self.init_iter = None
        self._sums = None

    def set_paths(self, data_path):
        """utils.add_config_paths: the files of one video under ``data_path``; creates the checkpoint folder."""
        self.video_path = os.path.join(data_path, "video")
        self.fg_masks_path = os.path.join(data_path, "masks")
        self.dino_embed_path = os.path.join(data_path, "dino_embeddings", "dino_embed_video.pt")
        self.fg_trajectories_path = os.path.join(data_path, "of_trajectories", "fg_trajectories.pt")
        self.bg_trajectories_path = os.path.join(data_path, "of_trajectories", "bg_trajectories.pt")
        self.dino_bb_path = os.path.join(data_path, "dino_best_buddies", "dino_best_buddies_filtered.pt")
        self.ckpt_folder = os.path.join(data_path, "models", "dino_tracker")
        os.makedirs(self.ckpt_folder, exist_ok=True)

    # ------------------------------------------------------------------ data
    def load_fg_masks(self):
        from .fg_masks import load_masks
        self.fg_masks = torch.from_numpy(load_masks(self.fg_masks_path, h_resize=self.config["video_resh"])).to(self.device)

    def load_dino_best_buddies(self):
        self.dino_bb_pairs = torch.load(self.dino_bb_path, map_location=self.device)

    def load_trajectories(self):
        assert os.path.exists(self.fg_trajectories_path) and os.path.exists(self.bg_trajectories_path), \
            "trajectory files don't exist"
        dev = torch.device("cpu") if self.config["keep_traj_in_cpu"] else self.device
        return (torch.load(self.fg_trajectories_path, map_location=dev),
                torch.load(self.bg_trajectories_path, map_location=dev))

    def get_sampler(self):
        from .sampler import DinoTrackerSampler
        fg, bg = self.load_trajectories()
        return DinoTrackerSampler(fg_trajectories=fg, bg_trajectories=bg, fg_traj_ratio=self.config["fg_traj_ratio"],
                                  batch_size=self.config["train_batch_size"], range_normalizer=self.range_normalizer,
                                  dst_range=(-1, 1), num_frames=self.config["batch_n_frames"],
                                  keep_in_cpu=self.config["keep_traj_in_cpu"])

    def get_model(self):
        """The tracker of this video with freshly initialised weights (dino_tracker.py:86-102)."""
        from .tracker import Tracker
        video = load_video(self.video_path, resize=(self.config["video_resh"], self.config["video_resw"])).to(self.device)
        cfg = self.config
        return Tracker(video=video, device=self.device, dino_embed_path=self.dino_embed_path,
                       dino_patch_size=cfg["dino_patch_size"], stride=cfg["stride"], ckpt_path=self.ckpt_folder,
                       cyc_n_frames=cfg["cyc_n_frames"], cyc_batch_size_per_frame=cfg["cyc_batch_size_per_frame"],
                       cyc_fg_points_ratio=cfg["cyc_fg_points_ratio"], cyc_thresh=cfg["cyc_thresh"])

    def train_setup(self):
        """dino_tracker.py:104-121: the model (checkpoint ``init_iter`` loaded when it is above 0), Adam over delta-DINO
        and the refiner, and the scheduler advanced ``init_iter`` steps."""
        model = self.get_model()
        self.init_iter = last_ckpt_iter(self.ckpt_folder)
        if self.init_iter > 0:
            model.load_weights(self.init_iter)
        optimizer = torch.optim.Adam([{"params": model.delta_dino.parameters(), "lr": self.config["lr_delta_dino"]},
                                      {"params": model.tracker_head.parameters(), "lr": self.config["lr_cnn_refiner"]}])
        scheduler = get_cnn_refiner_scheduler(optimizer, gamma=self.config["scheduler_gamma"],
                                              apply_every=self.config["apply_scheduler_every"])
        for _ in range(max(self.init_iter, 0)):
            scheduler.step()
        print("------- INIT ITER", self.init_iter)
        return model, optimizer, scheduler

    # ------------------------------------------------------------------ loss terms
    def tracking_loss(self, model, inputs, labels):
        return self.of_loss_fn(model(inputs), labels).mean()

    def cycle_loss(self, model, inputs):
        """dino_tracker.py:346-353."""
        cyc = model.get_cycle_consistent_preds(inputs[-1], self.fg_masks)
        weight = self.config["cyc_gamma"] ** cyc["cycle_consistency_dists"]
        st = weight[:, None] * self.of_loss_fn(cyc["source_target_coords"], cyc["target_coords"][:, :2])
        ts = weight[:, None] * self.of_loss_fn(cyc["target_source_coords"], cyc["source_coords"][:, :2])
        return (st.mean() + ts.mean()) / 2

    def refined_bb_loss(self, model, frames_set_t):
        from .contrastive import get_refined_bb_contrastive_loss
        cfg = self.config
        return get_refined_bb_contrastive_loss(self, model, frames_set_t, model.frame_embeddings,
                                               batch_size=cfg["cl_n_frames"], points_per_pair=cfg["cl_points_per_pair"],
                                               fg_points_ratio=cfg["cl_fg_points_ratio"], temp=cfg["cl_temp"],
                                               cl_div=cfg["cl_div_ref_bb"])

    def dino_bb_loss(self, model, frames_set_t):
        from .contrastive import get_dino_bb_contrastive_loss
        return get_dino_bb_contrastive_loss(self, model, frames_set_t)

    def regularisers(self, model):
        """(norm_reg, angle_reg) of the last forward's embeddings (dino_tracker.py:136-146)."""
        from .train import emb_regularisers
        return emb_regularisers(model)

    # ------------------------------------------------------------------ loop
    def iteration(self, i, model, sampler, optimizer, scheduler):
        """One iteration of dino_tracker.py:407-435.  Returns the detached loss terms in ``_TERMS`` order."""
        cfg = self.config
        optimizer.zero_grad()
        sample = sampler()
        labels = sample["t2_points_normalized"][:, :-1]
        inputs = (sample["t1_points"], sample["source_frame_indices"], sample["target_frame_indices"], sample["frames_set_t"])
        tracking_loss = self.tracking_loss(model, inputs, labels)
        # as in the reference, ``loss`` IS the tracking loss's tensor and the terms are added to it in place, so the
        # logged loss_of equals loss_total
        loss = tracking_loss
        zero = torch.zeros((), device=tracking_loss.device)
        cyc = ref = zero
        if i >= cfg.get("apply_cyc_after", 0):
            cyc = self.cycle_loss(model, inputs)
            loss += cfg["lambda_cyc"] * cyc
        if i >= cfg.get("apply_cl_ref_after", 0):
            ref = self.refined_bb_loss(model, inputs[-1])
            loss += cfg["lambda_cl_ref_bb"] * ref
        dino = self.dino_bb_loss(model, inputs[-1])
        norm_reg, angle_reg = self.regularisers(model)
        loss += cfg["lambda_cl_dino_bb"] * dino + cfg["lambda_emb_norm"] * norm_reg + cfg["lambda_angle"] * angle_reg
        loss.backward()
        optimizer.step()
        scheduler.step()
        return torch.stack([loss, tracking_loss, dino, ref, norm_reg, angle_reg, cyc]).detach()

    def log_losses(self, i):
        """dino_tracker.py:373-390: the running means over the last log interval (the sums divided by 100, as the
        reference divides them), one ``logging.info`` line."""
        m = dict(zip(self._TERMS, (self._sums / self.LOG_INTERVAL).tolist()))
        s = (f"loss_of: {m['loss_of']:.4f}, loss_cl_dino_bb: {m['loss_cl_dino_bb']:.4f}, "
             f"loss_emb_norm_reg: {m['loss_emb_norm_reg']:.4f}, loss_angle_reg: {m['loss_angle_reg']:.4f}")
        if i >= self.config.get("apply_cl_ref_after", 0):
            s += f", loss_cl_refiner: {m['loss_cl_refiner']:.4f}"
        if i >= self.config.get("apply_cyc_after", 0):
            s += f", loss_cyc: {m['loss_cyc']:.4f}"
        s += f", loss_total: {m['loss_total']:.4f}"
        logging.info(s)
        self._sums.zero_()

    def train(self):
        """dino_tracker.py:392-448."""
        cfg = self.config
        self.load_fg_masks()
        total_iterations = cfg["total_iterations"]
        checkpoint_interval = cfg["checkpoint_interval"]
        sampler_batch_iterations = cfg.get("sampler_batch_iterations", 100_000)
        self.load_dino_best_buddies()
        sampler = self.get_sampler()
        model, optimizer, scheduler = self.train_setup()
        model.train()
        self._sums = None
        for i in tqdm(range(self.init_iter, total_iterations)):
            terms = self.iteration(i, model, sampler, optimizer, scheduler)
            self._sums = terms if self._sums is None else self._sums + terms
            if i % self.LOG_INTERVAL == 0:
                self.log_losses(i)
            if i == total_iterations - 1 or i % checkpoint_interval == 0:
                model.save_weights(i)
            if i % sampler_batch_iterations == 0 and i > 0:
                print("Loading next batch", flush=True)
                sampler.load_next_batch()
        model.save_weights(total_iterations)
        return model


def main(argv=None):
    """train.py: ``--config``, ``--data-path``, ``--seed`` (default 2); seeds every generator first."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="./config/train.yaml", type=str)
    ap.add_argument("--data-path", default="./dataset/libby", type=str)
    ap.add_argument("--seed", default=2, type=int)
    args = ap.parse_args(argv)
    fix_random_seeds(args.seed)
    with open(args.config) as f:
        config = yaml.safe_load(f.read())
    DinoTrackerTrainer(config, args.data_path).train()


if __name__ == "__main__":
    main()
