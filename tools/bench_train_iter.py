"""The time of one whole training iteration (dino_tracker.py:405-435 after iteration 5000: the cycle term and both
contrastive terms active) at train.yaml's shape, with two sampler routes alternated in the same process:
  (a) ``oracle``: the plain-torch sampler of data/dataset.py (oracle/sampler.py), the route the reference's trainer runs;
  (b) ``library``: dino_tracker_b200.sampler.DinoTrackerSampler.

    python tools/bench_train_iter.py [--steps 20] [--warmup 3] [--out DIR]

Set-up: 50 frames of 476 x 854, C = 1024 seeded features, the shipped delta-DINO widths, Adam + LambdaLR as
``train_setup`` builds them, trajectories chained from smooth flows (as tools/bench_fg_mask.py builds them, about 1M)
split by a planted mask, and a best-buddies dict for every ordered frame pair.  The loop body is restated with the
library's Tracker and contrastive losses (the reference is not importable here); the norm and angle regularisers are the
reference's torch expressions.  Per route: the median ms per iteration, the median CUDA-event ms of each phase, and the
peak device memory above the set-up's.  The card's name, power limit and SM clock are read in the same run.  Prints one
JSON line (and writes it to DIR/bench_train_iter.json with --out).
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
PHASES = ("sampler", "forward", "cycle", "refined_loss", "dino_bb_loss", "regularisers", "backward", "optimiser")


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_iter needs a CUDA device")
    from dino_tracker_b200 import contrastive as c
    from dino_tracker_b200 import sampler as sm
    from oracle import sampler as osm
    dev = "cuda:0"
    info = card()
    model, opt, sched, tr, fg, bg, shapes = setup(dev)
    rn = osm.RangeNormalizer(shapes=shapes, device=dev)
    huber = torch.nn.HuberLoss(delta=1 / 32, reduction="none")
    kw = dict(batch_size=CFG["train_batch_size"], range_normalizer=rn, dst_range=(-1, 1), fg_trajectories=fg,
              bg_trajectories=bg, fg_traj_ratio=CFG["fg_traj_ratio"], num_frames=CFG["batch_n_frames"])
    samplers = {"oracle": osm.DinoTrackerSampler(**kw), "library": sm.DinoTrackerSampler(**kw)}
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()

    def iteration(sampler):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(PHASES) + 1)]
        torch.cuda.empty_cache()
        opt.zero_grad()
        ev[0].record()
        sample = sampler()
        labels = sample["t2_points_normalized"][:, :-1]
        inputs = (sample["t1_points"], sample["source_frame_indices"], sample["target_frame_indices"], sample["frames_set_t"])
        ev[1].record()
        loss = huber(model(inputs), labels).mean()
        ev[2].record()
        cyc = model.get_cycle_consistent_preds(inputs[-1], tr.fg_masks)
        wgt = CFG["cyc_gamma"] ** cyc["cycle_consistency_dists"]
        st = wgt[:, None] * huber(cyc["source_target_coords"], cyc["target_coords"][:, :2])
        ts = wgt[:, None] * huber(cyc["target_source_coords"], cyc["source_coords"][:, :2])
        loss = loss + CFG["lambda_cyc"] * (st.mean() + ts.mean()) / 2
        ev[3].record()
        ref_l = c.get_refined_bb_contrastive_loss(tr, model, inputs[-1], model.frame_embeddings,
                                                  batch_size=CFG["cl_n_frames"], points_per_pair=CFG["cl_points_per_pair"],
                                                  fg_points_ratio=CFG["cl_fg_points_ratio"], temp=CFG["cl_temp"],
                                                  cl_div=CFG["cl_div_ref_bb"])
        loss = loss + CFG["lambda_cl_ref_bb"] * ref_l
        ev[4].record()
        dino_l = c.get_dino_bb_contrastive_loss(tr, model, inputs[-1])
        ev[5].record()
        emb, raw = model.frame_embeddings, model.raw_embeddings
        norm_reg = (emb.norm(dim=1) / raw.norm(dim=1) - 1).abs().mean()
        angle_reg = (torch.einsum("bchw,bchw->bhw", emb, raw) / (emb.norm(dim=1) * raw.norm(dim=1)) - 1).abs().mean()
        loss = loss + CFG["lambda_cl_dino_bb"] * dino_l + CFG["lambda_emb_norm"] * norm_reg + CFG["lambda_angle"] * angle_reg
        ev[6].record()
        loss.backward()
        ev[7].record()
        opt.step()
        sched.step()
        ev[8].record()
        loss.item()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[-1]), [ev[i].elapsed_time(ev[i + 1]) for i in range(len(PHASES))]

    res = {r: {"total": [], "phases": [], "peak": 0} for r in samplers}
    for it in range(args.warmup + args.steps):
        for route, s in samplers.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            total, phases = iteration(s)
            if it >= args.warmup:
                res[route]["total"].append(total)
                res[route]["phases"].append(phases)
                res[route]["peak"] = max(res[route]["peak"], torch.cuda.max_memory_allocated() - base)
    out = {"what": "train_iteration", "T": shapes[2], "H": shapes[1], "W": shapes[0], "C": 1024, "batch": CFG["train_batch_size"],
           "n_fg": fg.shape[0], "n_bg": bg.shape[0], "steps": args.steps, "warmup": args.warmup, "card": info}
    for route, r in res.items():
        out[route] = {"ms_median": round(statistics.median(r["total"]), 2),
                      "ms_min": round(min(r["total"]), 2), "ms_max": round(max(r["total"]), 2),
                      "phases_ms_median": {p: round(statistics.median(x[i] for x in r["phases"]), 3) for i, p in enumerate(PHASES)},
                      "peak_extra_gib": round(r["peak"] / 2 ** 30, 3)}
    out["card_after"] = card()
    print(json.dumps(out), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_train_iter.json"), "w") as f:
            f.write(json.dumps(out) + "\n")


if __name__ == "__main__":
    main()
