"""Foreground masks and the fg / bg split on the GPU: the kernels against the reference's torch route on the same GPU.

    python tools/bench_fg_mask.py [--frames 50 300] [--reps 3] [--out DIR]

For each T: C = 1024 planted features of 67 x 121 = 8,107 tokens per frame (476 x 854 at stride 7), the time and
torch.cuda.max_memory_allocated of ``fg_masks`` and of the oracle's restatement of create_fg_mask.py (normalize, reshape,
torch.pca_lowrank(q=3, niter=20), projection, interpolate), and the kernels' read bandwidth from passes x M x C x 4
bytes against the H100 SXM's 3.35 TB/s.  Then the split of ~1M trajectories.  The card's name and power limit are read
in the same run.  Prints one JSON line per measurement (and writes them to DIR/bench_fg_mask.jsonl with --out).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PASSES = 1 + 1 + 20 + 1          # stats, start, 20 subspace iterations, projection


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        out = f"unknown ({e})"
    return out


def timed(fn, reps):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return min(times), (torch.cuda.max_memory_allocated() - base) / 2 ** 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[50, 300])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fg_mask needs a CUDA device")
    from dino_tracker_b200 import fg_masks as fgm
    from oracle import fg_masks as ofg
    from dino_tracker_b200.trajectories import chain_trajectories
    from oracle import trajectories as otr
    dev = "cuda:0"
    rows = []
    info = card()
    h, w, C = 67, 121, 1024
    for T in args.frames:
        feats, _ = ofg.planted_features(T, h, w, C, seed=T, noise=0.6, device=dev)
        M = T * h * w
        fgm.fg_masks(feats[:1], (476, 854))                      # warm-up: module load, cuSOLVER handles
        t_k, mem_k = timed(lambda: fgm.fg_masks(feats, (476, 854), fg_mask_threshold=0.6), args.reps)
        row = dict(what="fg_mask", T=T, M=M, C=C, kernels_s=round(t_k, 4), kernels_extra_gib=round(mem_k, 3),
                   read_tb_s=round(PASSES * M * C * 4 / t_k / 1e12, 3), passes=PASSES, card=info)
        try:
            ofg.get_fg_mask_from_pca(feats[:1], (476, 854))
            t_o, mem_o = timed(lambda: ofg.get_fg_mask_from_pca(feats, (476, 854), fg_mask_threshold=0.6), 1)
            row.update(oracle_s=round(t_o, 4), oracle_extra_gib=round(mem_o, 3), speedup=round(t_o / t_k, 2))
        except torch.cuda.OutOfMemoryError:
            row.update(oracle_s=None, oracle_extra_gib="out of memory")
        torch.cuda.empty_cache()
        print(json.dumps(row), flush=True)
        rows.append(row)
        del feats
        torch.cuda.empty_cache()
    # split: chained smooth flows at 476 x 854, T = 50 (about 1M trajectories with every start frame)
    T, H, W = 50, 476, 854
    fwd, bwd, _ = otr.stack_flows(otr.smooth_flows(T, H, W, seed=5, amplitude=3.0, device=dev), T)
    traj = chain_trajectories(fwd, bwd, None, 1.0, 2)
    _, masks = ofg.split_case_inputs(1, T, H, W, seed=6)
    masks = masks.to(dev)
    fgm.split_trajectories(traj, masks)
    t_k, _ = timed(lambda: fgm.split_trajectories(traj, masks), 5)
    t_o, _ = timed(lambda: (ofg.mask_filter(traj, masks), ofg.mask_filter(traj, masks, filter_bg=True)), 5)
    row = dict(what="split", N=traj.shape[0], T=T, kernels_s=round(t_k, 5), oracle_s=round(t_o, 5),
               speedup=round(t_o / t_k, 2), card=info)
    print(json.dumps(row), flush=True)
    rows.append(row)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_fg_mask.jsonl"), "w") as f:
            f.writelines(json.dumps(r) + "\n" for r in rows)


if __name__ == "__main__":
    main()
