"""BASELINE config 5: best-buddies all-pairs mutual NN over T frames' patch embeddings; pairs sharded over ranks.
  python tools/bench_bb.py --T 24                  (1 GPU)
  torchrun --nproc-per-node N tools/bench_bb.py    (N GPUs: features replicated, unordered pairs dealt round-robin)
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=24)
    ap.add_argument("--C", type=int, default=1024)
    a = ap.parse_args()
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = f"cuda:{local}"
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(dev))
    from dino_tracker_b200 import _lib
    from dino_tracker_b200.best_buddies import nearest_neighbours
    feats = bench.synth_video_features(a.T, a.C, dev, 99, 0.5)          # T x C x h x w, same on every rank (replicated)
    tpc = feats.permute(0, 2, 3, 1).reshape(a.T, bench.P, a.C).contiguous()
    norms = tpc.norm(dim=2).contiguous()
    del feats
    geom = _lib.make_geom(bench.H, bench.W)
    unordered = [(s, t) for s in range(a.T) for t in range(s + 1, a.T)]
    mine = unordered[rank::world]
    ordered = [p for (s, t) in mine for p in ((s, t), (t, s))]
    nearest_neighbours(tpc, norms, geom, ordered[:4])                    # warm-up
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    nn_idx, nn_cos = nearest_neighbours(tpc, norms, geom, ordered)
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    n_ordered = a.T * (a.T - 1)
    if rank == 0:
        s = ms.item() / 1000
        print(json.dumps({"config": f"best-buddies T={a.T} C={a.C} 854x476", "n_gpus": world, "ordered_pairs": n_ordered,
                          "seconds": s, "ordered_pairs_per_s": n_ordered / s,
                          "algorithmic_tflops": 2.0 * bench.P ** 2 * a.C * n_ordered / s / 1e12,
                          "note": "each ordered pair = one 8107x8107xC affinity GEMM (wgmma split-fp16) + top-2 epilogue + exact resolve"}))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
