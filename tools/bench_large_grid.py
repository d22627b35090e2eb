"""Inference and one training step on token grids beyond 128 x 128 tokens, next to the shipped frame size.

    python tools/bench_large_grid.py [--reps 7] [--out DIR]

Workloads (seeded synthetic features, the bench's sharp head):
  * ``ModelInference.infer`` at 1274 x 714 (101 x 181 = 18,281 tokens) and at 854 x 476 (67 x 121 = 8,107 tokens), T = 50,
    256 lattice query points at t = 0, C = 1024: median of --reps CUDA-event timings after two warm-up calls, then one
    profiled call for the per-class times, and the split of the anchor-phase maps between the exact window and the full
    map (``_lib.infer_stats``).
  * one training step at 1274 x 714: ``Tracker.forward`` with gradients on 512 points of a 4-frame set (cached
    embeddings, C = 1024) and the backward of the Huber loss, median of --reps.
The card's name, power limit and SM clocks are read in the same run.  Prints one JSON line (and writes it to
DIR/bench_large_grid.json with --out).
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

DEV = "cuda:0"


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def features(T, C, h, w, seed):
    """Smooth descriptor field shifted per frame plus noise, drawn on the device (bench.py's construction at any grid)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    pad = 8
    base = torch.randn(C, h + 2 * pad, w + 2 * pad, device=DEV, generator=g)
    sm = base.clone()
    sm[:, 1:-1, 1:-1] = base[:, 1:-1, 1:-1] * 0.5 + 0.125 * (base[:, :-2, 1:-1] + base[:, 2:, 1:-1] +
                                                             base[:, 1:-1, :-2] + base[:, 1:-1, 2:])
    cg = torch.Generator().manual_seed(seed)
    out = torch.empty(T, C, h, w, device=DEV)
    s = torch.zeros(2, dtype=torch.long)
    for t in range(T):
        if t:
            s = (s + torch.randint(-1, 2, (2,), generator=cg)).clamp(-3, 3)
        out[t] = sm[:, pad + s[0]: pad + s[0] + h, pad + s[1]: pad + s[1] + w]
    out += 0.25 * torch.randn(out.shape, device=DEV, generator=g)
    return out


def timed(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return ms


def bench_infer(H, W, reps):
    from bench_inputs import lattice, sharp_head
    from dino_tracker_b200 import ModelInference, Tracker, _lib
    from oracle.tracker import Geometry
    geo = Geometry(H=H, W=W)
    T, C, side = 50, 1024, 16
    feats = features(T, C, geo.h, geo.w, 1234)
    m = Tracker(video=torch.zeros(T, 3, H, W, device=DEV), dino_embed_video=feats, device=DEV,
                delta_channels=[3, 4, 4, 4, C])
    m.tracker_head.load_state_dict(sharp_head(0))
    mi = ModelInference(m, m.range_normalizer, 0.7, 0.6)
    q = lattice(side, side, H, W, 0, 30.0, 0).to(DEV)
    ms = timed(lambda: mi.infer(q), reps)
    _lib.profile_enable(True)
    _lib.profile_collect()
    mi.infer(q)
    torch.cuda.synchronize()
    prof = _lib.profile_collect()
    _lib.profile_enable(False)
    st = _lib.infer_stats()
    res = {"frame": f"{W}x{H}", "tokens": geo.P, "grid": f"{geo.h}x{geo.w}", "T": T, "C": C, "queries": side * side,
           "median_ms": round(statistics.median(ms), 3), "min_ms": round(min(ms), 3), "max_ms": round(max(ms), 3),
           "per_class_ms": {k: round(v[0], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][0])},
           "anchor_maps": st["anchor_maps"], "exact_window": st["exact_window"], "full_map": st["full_map"],
           "exact_window_share": round(st["exact_window"] / max(st["anchor_maps"], 1), 4), "pipeline": st["pipeline"],
           "coarse": st["coarse"]}
    del m, mi, feats
    torch.cuda.empty_cache()
    return res


def bench_train_step(H, W, reps):
    import torch.nn.functional as F

    from bench_inputs import sharp_head
    from dino_tracker_b200 import Tracker
    from oracle.tracker import Geometry
    geo = Geometry(H=H, W=W)
    T, C, B, N = 8, 1024, 512, 4
    feats = features(T, C, geo.h, geo.w, 99)
    m = Tracker(video=torch.zeros(T, 3, H, W, device=DEV), dino_embed_video=feats, device=DEV,
                delta_channels=[3, 4, 4, 4, C])
    m.tracker_head.load_state_dict(sharp_head(0))
    m.cache_refined_embeddings()
    g = torch.Generator().manual_seed(5)
    pts = (torch.rand(B, 3, generator=g) * torch.tensor([W - 1.0, H - 1.0, 0.0])).to(DEV)
    src, tgt = torch.randint(0, N, (B,), generator=g).to(DEV), torch.randint(0, N, (B,), generator=g).to(DEV)
    labels = (torch.rand(B, 2, generator=g) * 2 - 1).to(DEV)
    fs = torch.tensor([0, 2, 4, 6], dtype=torch.int32, device=DEV)

    def step():
        m.zero_grad(set_to_none=True)
        F.huber_loss(m((pts, src, tgt, fs)), labels, delta=1 / 32).backward()

    ms = timed(step, reps)
    return {"frame": f"{W}x{H}", "tokens": geo.P, "points": B, "frame_set": N, "C": C,
            "median_ms": round(statistics.median(ms), 3), "min_ms": round(min(ms), 3), "max_ms": round(max(ms), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_large_grid.py needs a CUDA device")
    sys.path.insert(0, ROOT)
    res = {"card": card(),
           "infer": [bench_infer(714, 1274, a.reps), bench_infer(476, 854, a.reps)],
           "train_step": bench_train_step(714, 1274, a.reps)}
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_large_grid.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
