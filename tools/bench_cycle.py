"""The cycle-consistency term of the training step (models/tracker.py:182-301, dino_tracker.py:346-353) at train.yaml's
shape: 476 x 854, C = 1024, a 4-frame set of a 50-frame video, 4 pairs x 256 points, foreground ratio 0.7, threshold 4,
a planted mask of 84,000 foreground pixels per frame.  Two routes alternated in one process:
  (a) ``per_pair``: the per-pair algorithm restated on the public get_point_predictions and torch.randperm
      (tests/test_cycle_gpu.py), the route before the batched term;
  (b) ``library``: Tracker.get_cycle_consistent_preds (dino_tracker_b200/cycle.py).
Per route the median CUDA-event ms of the term's forward and of its share of the backward (the cycle loss alone,
backpropagated to the frame set's embeddings and the refiner), and on their own the four pairs' host draws: randperm
prefixes against torch.randperm at the mask's sizes.  The card's name, power limit and SM clock are read in the same run.

    python tools/bench_cycle.py [--steps 20] [--warmup 3] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cycle needs a CUDA device")
    from bench_train_iter import card
    from test_cycle_gpu import _cycle_loss, _reference_preds
    from test_delta_train_gpu import SHIPPED, _sd
    from dino_tracker_b200 import Tracker
    from dino_tracker_b200 import cycle
    from oracle import synth
    dev = "cuda:0"
    info = card()
    H, W, T, C = 476, 854, 50, 1024
    h, w = (H - 14) // 7 + 1, (W - 14) // 7 + 1
    m = Tracker(video=synth.random_video(T, H, W, seed=401).to(dev), dino_embed_video=synth.random_features(T, C, h, w, seed=400),
                device=dev, delta_channels=SHIPPED)
    m.tracker_head.load_state_dict(synth.head_weights("well", seed=402))
    m.delta_dino.load_state_dict(_sd(SHIPPED, 403, last_std=0.02))
    m.train()
    fg = torch.zeros(T, H, W, device=dev)
    fg[:, 120:360, 250:600] = 1
    n_fg = int(fg[0].sum())
    g = torch.Generator().manual_seed(404)
    B = 512
    fs = torch.randperm(T, generator=g)[:4].sort().values.to(dev)
    inp = ((torch.rand(B, 3, generator=g) * torch.tensor([W - 1.0, H - 1.0, 0.0])).to(dev),
           torch.randint(0, 4, (B,), generator=g).to(dev), torch.randint(0, 4, (B,), generator=g).to(dev), fs)
    params = list(m.delta_dino.parameters()) + list(m.tracker_head.parameters())
    routes = {"per_pair": lambda: _reference_preds(m, fs, fg)[1], "library": lambda: m.get_cycle_consistent_preds(fs, fg)}

    def once(fn):
        m(inp)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        torch.cuda.synchronize()
        ev[0].record()
        loss = _cycle_loss(fn())
        ev[1].record()
        torch.autograd.grad(loss, params, allow_unused=True)
        ev[2].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), loss.item()

    res = {r: {"fwd": [], "bwd": []} for r in routes}
    for it in range(args.warmup + args.steps):
        for r, fn in routes.items():
            torch.manual_seed(1000 + it)
            f, b, _ = once(fn)
            if it >= args.warmup:
                res[r]["fwd"].append(f)
                res[r]["bwd"].append(b)
    # the host draws of one iteration (4 pairs: a foreground and a background randperm each), on their own
    draws = {}
    for name, fn in (("torch_randperm", lambda n, k: torch.randperm(n)[:k]), ("prefix", cycle.randperm_prefix)):
        ts = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            for _ in range(4):
                fn(n_fg, 179)
                fn(H * W - n_fg, 77)
            ts.append((time.perf_counter() - t0) * 1e3)
        draws[name] = round(statistics.median(ts), 3)
    out = {"what": "cycle_term", "H": H, "W": W, "C": C, "pairs": 4, "points_per_pair": 256, "n_fg": n_fg,
           "steps": args.steps, "warmup": args.warmup, "card": info, "host_draws_ms_median": draws}
    for r, v in res.items():
        out[r] = {"forward_ms_median": round(statistics.median(v["fwd"]), 3),
                  "backward_ms_median": round(statistics.median(v["bwd"]), 3)}
    out["card_after"] = card()
    print(json.dumps(out), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_cycle.json"), "w") as f:
            f.write(json.dumps(out) + "\n")


if __name__ == "__main__":
    main()
