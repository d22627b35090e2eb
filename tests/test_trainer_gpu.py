"""The native trainer (dino_tracker_b200/trainer.py) on the GPU.

* One iteration forced to the same weights and generator states: ``DinoTrackerTrainer.iteration`` (library sampler,
  regulariser node) against the reference's loop body (dino_tracker.py:407-429) restated here with the plain-torch
  sampler of data/dataset.py (oracle/sampler.py) and the reference's torch regulariser expressions, everything else from
  the library; before and after both apply thresholds.  Bars: identical generator states after the step; every loss term
  within 1e-6 relative; gradients within 2e-3 of each tensor's largest entry (the training-step bar of
  test_train_gpu.py; a convolution bias in front of a train-mode BatchNorm, whose gradient is 0 up to rounding, against
  that BatchNorm's gamma and beta gradients); parameters after the Adam step within 2e-3 of the step's largest change,
  on the entries whose gradient is above that bar (Adam's first step moves each entry by lr * sign(g), so the direction
  of an entry whose gradient is within the bar of 0 is not determined by the gradient bar).
* End to end from a folder in the reference's layout through the command-line entry: checkpoint names and keys, the
  checkpoints load into a Tracker that ``ModelInference.infer`` runs on, and a second run resumes from the last one.
"""
import copy
import os

import numpy as np
import pytest
import torch
import yaml
from PIL import Image

from oracle import contrastive as oc
from oracle import delta_dino as od
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REL = 1e-6
GRAD_TOL = 2e-3
# train.yaml's values, scaled down to a 6-frame 112 x 854 video (854 wide: masks load at the reference's default width)
H, W, T, C = 112, 854, 6, 32
CONFIG = {"checkpoint_interval": 2, "video_resw": W, "video_resh": H, "fg_traj_ratio": 0.5, "keep_traj_in_cpu": False,
          "train_batch_size": 64, "batch_n_frames": 4, "total_iterations": 4, "lr_delta_dino": 0.01, "lr_cnn_refiner": 0.01,
          "apply_scheduler_every": 2, "scheduler_gamma": 0.999, "lambda_cyc": 0.5, "apply_cyc_after": 5, "cyc_n_frames": 4,
          "cyc_batch_size_per_frame": 32, "cyc_fg_points_ratio": 0.7, "cyc_thresh": 4, "cyc_gamma": 0.8,
          "lambda_emb_norm": 0.0001, "lambda_angle": 0.0001, "lambda_cl_dino_bb": 0.00025, "lambda_cl_ref_bb": 0.00005,
          "cl_n_frames": 4, "cl_points_per_pair": 32, "cl_fg_points_ratio": 0.7, "cl_temp": 0.1, "cl_div_dino_bb": 700,
          "cl_div_ref_bb": 900, "apply_cl_ref_after": 5, "bb_amb_sig_a": 27, "bb_amb_sig_b": -5.7, "stride": 7,
          "dino_patch_size": 14, "anchor_cosine_similarity_threshold": 0.7, "cosine_similarity_threshold": 0.6}
FG_BOX = (30, 90, 250, 600)   # y0, y1, x0, x1 of the foreground


def _write_dataset(root, seed=0):
    """A video folder in the reference's layout (utils.add_config_paths): frames, masks, fg / bg trajectories, DINO
    embeddings and a filtered best-buddies dict for every ordered frame pair."""
    g = torch.Generator().manual_seed(seed)
    for d in ("video", "masks", "of_trajectories", "dino_embeddings", "dino_best_buddies"):
        os.makedirs(os.path.join(root, d), exist_ok=True)
    y0, y1, x0, x1 = FG_BOX
    for t in range(T):
        frame = (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8).numpy()
        Image.fromarray(frame).save(os.path.join(root, "video", f"{t:05d}.png"))
        mask = np.zeros((H, W), np.uint8)
        mask[y0:y1, x0:x1] = 255
        Image.fromarray(mask).save(os.path.join(root, "masks", f"{t:05d}.png"))

    def trajectories(n, inside):
        start = torch.rand(n, 2, generator=g)
        if inside:
            start = start * torch.tensor([x1 - x0 - 20.0, y1 - y0 - 10.0]) + torch.tensor([x0 + 5.0, y0 + 2.0])
        else:
            start = start * torch.tensor([x0 - 20.0, H - 10.0]) + 5.0
        steps = torch.arange(T, dtype=torch.float32)[None, :, None] * torch.tensor([1.5, 0.5])
        traj = start[:, None, :] + steps
        traj[: n // 4, T - 1] = float("nan")          # some trajectories end early
        return traj
    torch.save(trajectories(400, True), os.path.join(root, "of_trajectories", "fg_trajectories.pt"))
    torch.save(trajectories(400, False), os.path.join(root, "of_trajectories", "bg_trajectories.pt"))
    h, w = (H - 14) // 7 + 1, (W - 14) // 7 + 1
    torch.save(synth.random_features(T, C, h, w, seed=seed + 1), os.path.join(root, "dino_embeddings", "dino_embed_video.pt"))
    coords = oc.get_vit_feature_coords_from_mask(H, W, 7, 14)
    bb = {}
    for s in range(T):
        for t in range(T):
            if s != t:
                n = 120
                bb[f"{s}_{t}"] = {"source_coords": coords[torch.randperm(h * w, generator=g)[:n]],
                                  "target_coords": coords[torch.randint(h * w, (n,), generator=g)],
                                  "cos_sims": torch.rand(n, generator=g) * 0.6 + 0.4, "r": torch.rand(n, generator=g) * 0.4}
    torch.save(bb, os.path.join(root, "dino_best_buddies", "dino_best_buddies_filtered.pt"))
    return root


def _trainer(root, **overrides):
    from dino_tracker_b200.trainer import DinoTrackerTrainer
    tr = DinoTrackerTrainer(dict(CONFIG, **overrides), root, device=DEV)
    tr.load_fg_masks()
    tr.load_dino_best_buddies()
    return tr


def _reference_body(tr, i, model, sampler, optimizer, scheduler):
    """dino_tracker.py:407-429 with the plain-torch sampler and the reference's regularisers as torch expressions."""
    from dino_tracker_b200 import contrastive as c
    cfg = tr.config
    optimizer.zero_grad()
    sample = sampler()
    labels = sample["t2_points_normalized"][:, :-1]
    inputs = (sample["t1_points"], sample["source_frame_indices"], sample["target_frame_indices"], sample["frames_set_t"])
    tracking_loss = tr.of_loss_fn(model(inputs), labels).mean()
    loss = tracking_loss
    zero = torch.zeros((), device=DEV)
    cyc = ref = zero
    if i >= cfg["apply_cyc_after"]:
        p = model.get_cycle_consistent_preds(inputs[-1], tr.fg_masks)
        wgt = cfg["cyc_gamma"] ** p["cycle_consistency_dists"]
        st = wgt[:, None] * tr.of_loss_fn(p["source_target_coords"], p["target_coords"][:, :2])
        ts = wgt[:, None] * tr.of_loss_fn(p["target_source_coords"], p["source_coords"][:, :2])
        cyc = (st.mean() + ts.mean()) / 2
        loss += cfg["lambda_cyc"] * cyc
    if i >= cfg["apply_cl_ref_after"]:
        ref = c.get_refined_bb_contrastive_loss(tr, model, inputs[-1], model.frame_embeddings, batch_size=cfg["cl_n_frames"],
                                                points_per_pair=cfg["cl_points_per_pair"],
                                                fg_points_ratio=cfg["cl_fg_points_ratio"], temp=cfg["cl_temp"],
                                                cl_div=cfg["cl_div_ref_bb"])
        loss += cfg["lambda_cl_ref_bb"] * ref
    dino = c.get_dino_bb_contrastive_loss(tr, model, inputs[-1])
    emb, raw = model.frame_embeddings, model.raw_embeddings
    norm_reg = (emb.norm(dim=1) / raw.norm(dim=1) - 1).abs().mean()
    angle_reg = (torch.einsum("bchw,bchw->bhw", emb, raw) / (emb.norm(dim=1) * raw.norm(dim=1)) - 1).abs().mean()
    loss += cfg["lambda_cl_dino_bb"] * dino + cfg["lambda_emb_norm"] * norm_reg + cfg["lambda_angle"] * angle_reg
    loss.backward()
    optimizer.step()
    scheduler.step()
    return torch.stack([loss, tracking_loss, dino, ref, norm_reg, angle_reg, cyc]).detach()


def _run(tr, model, state, rng, body, sampler, i):
    model.load_state_dict(state)
    tr.get_model = lambda: model
    _, optimizer, scheduler = tr.train_setup()
    model.train()
    torch.set_rng_state(rng[0])
    torch.cuda.set_rng_state(rng[1])
    terms = body(i, model, sampler, optimizer, scheduler)
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    params = {k: p.detach().clone() for k, p in model.named_parameters()}
    return terms.cpu(), grads, params, (torch.get_rng_state(), torch.cuda.get_rng_state())


def _grad_scale(grads, k):
    """The largest entry of gradient k; for a convolution bias in front of a train-mode BatchNorm (mathematically 0, its
    computed gradient is rounding noise) that of the BatchNorm's gamma and beta, as test_delta_train_gpu.py bars it."""
    for ci, bi in zip(od.CONV_IDX, od.BN_IDX):
        if k == f"delta_dino.layers.{ci}.bias":
            return max(grads[f"delta_dino.layers.{bi}.weight"].abs().max().item(),
                       grads[f"delta_dino.layers.{bi}.bias"].abs().max().item())
    return grads[k].abs().max().item()


@pytest.mark.parametrize("i", [0, 5], ids=["before_thresholds", "after_thresholds"])
def test_iteration_matches_reference_body(tmp_path, i):
    from dino_tracker_b200 import sampler as sm
    from oracle import sampler as osm
    tr = _trainer(_write_dataset(str(tmp_path)))
    model = tr.get_model()
    chans = model.delta_dino.channels
    model.delta_dino.load_state_dict(od.random_state_dict(chans, torch.Generator().manual_seed(7), last_std=0.3))
    model.tracker_head.load_state_dict(synth.head_weights("well", seed=8))
    state = copy.deepcopy(model.state_dict())
    p0 = {k: p.detach().clone() for k, p in model.named_parameters()}
    fg, bg = tr.load_trajectories()
    rn = osm.RangeNormalizer(shapes=(W, H, T), device=DEV)
    kw = dict(batch_size=CONFIG["train_batch_size"], range_normalizer=rn, dst_range=(-1, 1), fg_trajectories=fg,
              bg_trajectories=bg, fg_traj_ratio=CONFIG["fg_traj_ratio"], num_frames=CONFIG["batch_n_frames"])
    lib_sampler, ref_sampler = sm.DinoTrackerSampler(**kw), osm.DinoTrackerSampler(**kw)
    torch.manual_seed(100 + i)
    rng = (torch.get_rng_state(), torch.cuda.get_rng_state())
    t_a, g_a, p_a, rng_a = _run(tr, model, state, rng, tr.iteration, lib_sampler, i)
    t_b, g_b, p_b, rng_b = _run(tr, model, state, rng, lambda *a: _reference_body(tr, *a), ref_sampler, i)
    assert torch.equal(rng_a[0], rng_b[0]) and torch.equal(rng_a[1], rng_b[1]), "different random draws"
    active = {0: (0, 1, 2, 4, 5), 5: (0, 1, 2, 3, 4, 5, 6)}[i]
    for k in range(7):
        if k in active:
            assert t_b[k] != 0 and abs(t_a[k] - t_b[k]) <= REL * abs(t_b[k]), (k, t_a[k].item(), t_b[k].item())
        else:
            assert t_a[k] == 0 and t_b[k] == 0
    for k in g_b:
        scale = _grad_scale(g_b, k)
        assert (g_a[k] - g_b[k]).abs().max().item() <= GRAD_TOL * scale, k
        step = (p_b[k] - p0[k]).abs().max().item()
        sure = g_b[k].abs() > GRAD_TOL * scale
        if sure.any():
            assert (p_a[k] - p_b[k])[sure].abs().max().item() <= GRAD_TOL * step, k


def test_cli_trains_writes_checkpoints_and_resumes(tmp_path, capsys):
    from dino_tracker_b200 import ModelInference, Tracker
    from dino_tracker_b200.trainer import main
    root = _write_dataset(str(tmp_path / "video"))
    cfg = str(tmp_path / "train.yaml")
    with open(cfg, "w") as f:
        yaml.safe_dump(CONFIG, f)
    main(["--config", cfg, "--data-path", root, "--seed", "2"])
    folder = os.path.join(root, "models", "dino_tracker")
    # fresh folder: iterations -1 .. 3, checkpoints at i % 2 == 0, at total - 1 and at total
    want = {f"{n}_{k}.pt" for n in ("tracker_head", "delta_dino") for k in (0, 2, 3, 4)}
    assert set(os.listdir(folder)) == want
    video = torch.zeros(T, 3, H, W, device=DEV)
    fresh = Tracker(video=video, dino_embed_path=os.path.join(root, "dino_embeddings", "dino_embed_video.pt"), device=DEV,
                    ckpt_path=folder)
    for k in (0, 2, 3, 4):
        assert set(torch.load(os.path.join(folder, f"tracker_head_{k}.pt"))) == set(fresh.tracker_head.state_dict())
        assert set(torch.load(os.path.join(folder, f"delta_dino_{k}.pt"))) == set(fresh.delta_dino.state_dict())
    fresh.load_weights(4)
    trained = torch.load(os.path.join(folder, "tracker_head_4.pt"))
    assert all(torch.equal(v.cpu(), trained[k].cpu()) for k, v in fresh.tracker_head.state_dict().items())
    q = synth.lattice_query_points(3, 2, H, W, t_q=[0, 1, 2, 3, 4, 5], margin=30.0, jitter_seed=1).to(DEV)
    with torch.no_grad():
        fresh.cache_refined_embeddings()
        traj, occ = ModelInference(fresh, fresh.range_normalizer, CONFIG["anchor_cosine_similarity_threshold"],
                                   CONFIG["cosine_similarity_threshold"]).infer(q)
    assert traj.shape == (q.shape[0], T, 2) and occ.shape == (q.shape[0], T) and torch.isfinite(traj).all()
    capsys.readouterr()
    cfg2 = str(tmp_path / "train6.yaml")
    with open(cfg2, "w") as f:
        yaml.safe_dump(dict(CONFIG, total_iterations=6), f)
    main(["--config", cfg2, "--data-path", root, "--seed", "2"])
    assert "------- INIT ITER 4" in capsys.readouterr().out
    assert set(os.listdir(folder)) == want | {f"{n}_{k}.pt" for n in ("tracker_head", "delta_dino") for k in (5, 6)}
