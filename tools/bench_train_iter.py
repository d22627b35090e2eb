"""The time of one whole training iteration (dino_tracker.py:405-435 after iteration 5000: the cycle term and both
contrastive terms active) at train.yaml's shape: ``DinoTrackerTrainer.iteration`` (dino_tracker_b200/trainer.py), three
routes alternated in the same process:
  (a) ``trainer``: the trainer as it ships (library sampler, the regulariser node);
  (b) ``trainer_torch_reg``: the trainer with the reference's torch regulariser expressions in place of the node;
  (c) ``oracle_sampler``: the trainer with the plain-torch sampler of data/dataset.py (oracle/sampler.py), the sampler
      the reference's trainer runs.
Then the two regularisers on their own on the frame set's embeddings (4 x 1024 x 67 x 121, token-major as the training
forward leaves them): the node's forward and backward against the torch expressions' forward and backward.

    python tools/bench_train_iter.py [--steps 20] [--warmup 3] [--reg-reps 50] [--out DIR]

Set-up: 50 frames of 476 x 854, C = 1024 seeded features, the shipped delta-DINO widths, Adam + LambdaLR as
``train_setup`` builds them, trajectories chained from smooth flows (as tools/bench_fg_mask.py builds them, about 1M)
split by a planted mask, and a best-buddies dict for every ordered frame pair.  Per route: the median ms per iteration
and the peak device memory above the set-up's; per regulariser implementation the median CUDA-event ms of forward and
backward.  The card's name, power limit and SM clock are read in the same run.  Prints one JSON line (and writes it to
DIR/bench_train_iter.json with --out).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CFG = {"lr_delta_dino": 0.01, "lr_cnn_refiner": 0.01, "scheduler_gamma": 0.999, "apply_scheduler_every": 40,
       "lambda_cyc": 0.5, "cyc_gamma": 0.8, "lambda_emb_norm": 0.0001, "lambda_angle": 0.0001, "lambda_cl_dino_bb": 0.00025,
       "lambda_cl_ref_bb": 0.00005, "cl_n_frames": 4, "cl_points_per_pair": 256, "cl_fg_points_ratio": 0.7, "cl_temp": 0.1,
       "cl_div_dino_bb": 700, "cl_div_ref_bb": 900, "bb_amb_sig_a": 27, "bb_amb_sig_b": -5.7, "dino_patch_size": 14,
       "train_batch_size": 512, "batch_n_frames": 4, "fg_traj_ratio": 0.5}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def setup(dev):
    from test_delta_train_gpu import SHIPPED, _sd
    from dino_tracker_b200 import Tracker
    from dino_tracker_b200.fg_masks import split_trajectories
    from dino_tracker_b200.trajectories import chain_trajectories
    from oracle import contrastive as oc
    from oracle import synth
    from oracle import trajectories as otr
    H, W, T, C = 476, 854, 50, 1024
    h, w = (H - 14) // 7 + 1, (W - 14) // 7 + 1
    feats = synth.random_features(T, C, h, w, seed=400)
    video = synth.random_video(T, H, W, seed=401).to(dev)
    model = Tracker(video=video, dino_embed_video=feats, device=dev, delta_channels=SHIPPED)
    model.tracker_head.load_state_dict(synth.head_weights("well", seed=402))
    model.delta_dino.load_state_dict(_sd(SHIPPED, 403, last_std=0.02))
    model.train()
    params = [{"params": model.delta_dino.parameters(), "lr": CFG["lr_delta_dino"]},
              {"params": model.tracker_head.parameters(), "lr": CFG["lr_cnn_refiner"]}]
    opt = torch.optim.Adam(params)
    gamma, every = CFG["scheduler_gamma"], CFG["apply_scheduler_every"]
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lr_lambda=[lambda e: gamma ** (e // every), lambda e: 1])
    fwd, bwd, _ = otr.stack_flows(otr.smooth_flows(T, H, W, seed=5, amplitude=3.0, device=dev), T)
    traj = chain_trajectories(fwd, bwd, None, 1.0, 2)
    del fwd, bwd
    fg_masks = torch.zeros(T, H, W, device=dev)
    fg_masks[:, 120:360, 250:600] = 1
    fg, bg = split_trajectories(traj, (fg_masks > 0).to(torch.uint8))
    del traj
    g = torch.Generator().manual_seed(404)
    coords = oc.get_vit_feature_coords_from_mask(H, W, 7, 14)
    bb = {}
    for s in range(T):
        for t in range(T):
            if s != t:
                n = 300
                bb[f"{s}_{t}"] = {"source_coords": coords[torch.randperm(h * w, generator=g)[:n]].to(dev),
                                  "target_coords": coords[torch.randint(h * w, (n,), generator=g)].to(dev),
                                  "cos_sims": (torch.rand(n, generator=g) * 0.6 + 0.4).to(dev),
                                  "r": (torch.rand(n, generator=g) * 0.4).to(dev)}
    tr = type("Trainer", (), {})()
    tr.config, tr.fg_masks, tr.dino_bb_pairs = CFG, fg_masks, bb
    return model, opt, sched, tr, fg, bg, (W, H, T)


def torch_regularisers(model):
    """dino_tracker.py:136-146 as the reference evaluates them."""
    emb, raw = model.frame_embeddings, model.raw_embeddings
    norm_reg = (emb.norm(dim=1) / raw.norm(dim=1) - 1).abs().mean()
    angle_reg = (torch.einsum("bchw,bchw->bhw", emb, raw) / (emb.norm(dim=1) * raw.norm(dim=1)) - 1).abs().mean()
    return norm_reg, angle_reg


def trainer_for(tr_stub, T, workdir):
    """A DinoTrackerTrainer over the set-up's masks and best buddies (its data folder holds only T placeholder frames:
    the trainer reads the frame count from it)."""
    from PIL import Image
    from dino_tracker_b200.trainer import DinoTrackerTrainer
    os.makedirs(os.path.join(workdir, "video"))
    for t in range(T):
        Image.new("RGB", (1, 1)).save(os.path.join(workdir, "video", f"{t:05d}.png"))
    cfg = dict(CFG, video_resw=854, video_resh=476)
    tr = DinoTrackerTrainer(cfg, workdir, device="cuda:0")
    tr.fg_masks, tr.dino_bb_pairs = tr_stub.fg_masks, tr_stub.dino_bb_pairs
    return tr


def time_regularisers(reps):
    """ms (median of reps) of the node's and the torch expressions' forward and backward on 4 x 1024 x 67 x 121."""
    from oracle import synth
    from dino_tracker_b200.train import RegularisersFunction, token_rows
    n, C, h, w = 4, 1024, 67, 121
    raw = synth.random_features(n, C, h, w, seed=410).cuda().permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    emb = (raw * 1.05 + 0.01 * torch.randn_like(raw)).requires_grad_(True)
    g = torch.ones((), device="cuda:0")

    def node():
        return RegularisersFunction.apply(token_rows(emb), token_rows(raw))

    def ref():
        class M:
            frame_embeddings, raw_embeddings = emb, raw
        return torch_regularisers(M)
    out = {}
    for name, fn in (("node", node), ("torch", ref)):
        fwd, bwd = [], []
        for r in range(reps + 3):
            emb.grad = None
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
            a, b = fn()
            ev[1].record()
            torch.autograd.backward([a, b], [g, g])
            ev[2].record()
            torch.cuda.synchronize()
            if r >= 3:
                fwd.append(ev[0].elapsed_time(ev[1]))
                bwd.append(ev[1].elapsed_time(ev[2]))
        out[name] = {"forward_ms": round(statistics.median(fwd), 4), "backward_ms": round(statistics.median(bwd), 4)}
    # what the node must move at least: forward reads E and R, backward reads both and writes dE
    nbytes = n * C * h * w * 4
    out["min_bytes"] = {"forward": 2 * nbytes, "backward": 3 * nbytes}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reg-reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_iter needs a CUDA device")
    import tempfile
    from dino_tracker_b200 import sampler as sm
    from oracle import sampler as osm
    dev = "cuda:0"
    info = card()
    model, opt, sched, stub, fg, bg, shapes = setup(dev)
    rn = osm.RangeNormalizer(shapes=shapes, device=dev)
    kw = dict(batch_size=CFG["train_batch_size"], range_normalizer=rn, dst_range=(-1, 1), fg_trajectories=fg,
              bg_trajectories=bg, fg_traj_ratio=CFG["fg_traj_ratio"], num_frames=CFG["batch_n_frames"])
    library, oracle_sampler = sm.DinoTrackerSampler(**kw), osm.DinoTrackerSampler(**kw)
    with tempfile.TemporaryDirectory() as workdir:
        tr = trainer_for(stub, shapes[2], workdir)
    node_reg = tr.regularisers
    routes = {"trainer": (library, node_reg), "trainer_torch_reg": (library, torch_regularisers),
              "oracle_sampler": (oracle_sampler, node_reg)}
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()

    def iteration(sampler, regularisers):
        tr.regularisers = regularisers
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        terms = tr.iteration(6000, model, sampler, opt, sched)
        ev[1].record()
        terms.tolist()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1])

    res = {r: {"total": [], "peak": 0} for r in routes}
    for it in range(args.warmup + args.steps):
        for route, (s, reg) in routes.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            total = iteration(s, reg)
            if it >= args.warmup:
                res[route]["total"].append(total)
                res[route]["peak"] = max(res[route]["peak"], torch.cuda.max_memory_allocated() - base)
    out = {"what": "train_iteration", "T": shapes[2], "H": shapes[1], "W": shapes[0], "C": 1024, "batch": CFG["train_batch_size"],
           "n_fg": fg.shape[0], "n_bg": bg.shape[0], "steps": args.steps, "warmup": args.warmup, "card": info}
    for route, r in res.items():
        out[route] = {"ms_median": round(statistics.median(r["total"]), 2),
                      "ms_min": round(min(r["total"]), 2), "ms_max": round(max(r["total"]), 2),
                      "peak_extra_gib": round(r["peak"] / 2 ** 30, 3)}
    del model, opt, sched, library, oracle_sampler, tr
    torch.cuda.empty_cache()
    out["regularisers"] = time_regularisers(args.reg_reps)
    out["card_after"] = card()
    print(json.dumps(out), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_train_iter.json"), "w") as f:
            f.write(json.dumps(out) + "\n")


if __name__ == "__main__":
    main()
