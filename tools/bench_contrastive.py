"""Time the best-buddy contrastive losses of the training step at train.yaml's shape (4 frames of 476 x 854, C = 1024,
4 pairs x 256 points, tau = 0.1): the library's drop-in losses (dino_tracker_b200/contrastive.py) against the plain-torch
losses (oracle/contrastive.py, fp32 at torch's default TF32 setting), forward + backward, alternating the two, medians of
--repeats after a warm-up of every shape.  The refined loss's in-training search and its InfoNCE node are also timed on
their own.  Prints one JSON line with the card, its power limit and the SM clock sampled in the same run.

    python tools/bench_contrastive.py [--repeats 7] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from dino_tracker_b200 import contrastive as cl  # noqa: E402
from oracle import contrastive as oc  # noqa: E402

CFG = {"cl_n_frames": 4, "cl_points_per_pair": 256, "cl_fg_points_ratio": 0.7, "cl_temp": 0.1, "cl_div_dino_bb": 700,
       "cl_div_ref_bb": 900, "bb_amb_sig_a": 27, "bb_amb_sig_b": -5.7, "dino_patch_size": 14}
H, W, C, N, T = 476, 854, 1024, 4, 8


def gpu_info():
    q = "name,power.limit,clocks.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def inputs(dev):
    g = torch.Generator().manual_seed(0)
    h, w = (H - 14) // 7 + 1, (W - 14) // 7 + 1
    yy, xx = torch.meshgrid(torch.arange(h).float(), torch.arange(w).float(), indexing="ij")
    freq = torch.rand(C, 2, generator=g) * 0.3
    phase = torch.rand(C, generator=g) * 6.28
    emb = torch.stack([torch.sin(freq[:, 0, None, None] * (xx + 1.3 * i) + freq[:, 1, None, None] * yy + phase[:, None, None])
                       + 0.05 * torch.randn(C, h, w, generator=g) for i in range(N)]).to(dev)
    masks = torch.zeros(T, H, W, device=dev)
    masks[:, 120:360, 250:600] = 1
    coords = oc.get_vit_feature_coords_from_mask(H, W, 7, 14)
    bb = {}
    for s in range(T):
        for t in range(T):
            if s != t:
                n = 2000
                bb[f"{s}_{t}"] = {"source_coords": coords[torch.randperm(h * w, generator=g)[:n]].to(dev),
                                  "target_coords": coords[torch.randint(h * w, (n,), generator=g)].to(dev),
                                  "cos_sims": (torch.rand(n, generator=g) * 0.6 + 0.4).to(dev),
                                  "r": (torch.rand(n, generator=g) * 0.4).to(dev)}
    tr = type("Trainer", (), {})()
    tr.config, tr.fg_masks, tr.dino_bb_pairs = CFG, masks, bb
    return tr, emb


def timed(fn, dev):
    torch.cuda.synchronize(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize(dev)
    return a.elapsed_time(b), (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_contrastive: needs a CUDA device")
    dev = torch.device("cuda")
    tr, emb0 = inputs(dev)
    fs = torch.arange(N, device=dev)
    video = torch.zeros(1, 3, H, W)

    def loss_fn(impl, which):
        def run():
            emb = emb0.clone().requires_grad_(True)
            model = oc.ModelStandIn(video, emb)
            torch.manual_seed(0)
            if which == "dino":
                loss = impl.get_dino_bb_contrastive_loss(tr, model, fs)
            else:
                loss = impl.get_refined_bb_contrastive_loss(tr, model, fs, emb, CFG["cl_n_frames"], CFG["cl_points_per_pair"],
                                                            CFG["cl_fg_points_ratio"], CFG["cl_temp"], CFG["cl_div_ref_bb"])
            loss.backward()
        return run

    pairs = [(0, 1), (2, 2), (3, 0), (1, 3)]

    def search():
        cl.refined_best_buddies(emb0, pairs, H, W)

    def infonce():
        E = cl._token_rows(emb0).contiguous().requires_grad_(True)
        P = E.shape[1]
        idx = torch.arange(256, device=dev) * 29
        rows = E.reshape(-1, C)
        src = torch.cat([s * P + idx for s, _ in pairs])
        tgt = torch.cat([t * P + idx + 3 for _, t in pairs])
        groups = [(s, t, 256 * k, 256) for k, (s, t) in enumerate(pairs)]
        cl1, cl2, _, _ = cl.bb_contrastive(E, rows[src], rows[tgt], groups, CFG["cl_temp"])
        (cl1.sum() + cl2.sum()).backward()

    cases = {"refined_lib": loss_fn(cl, "refined"), "refined_torch": loss_fn(oc, "refined"),
             "dino_bb_lib": loss_fn(cl, "dino"), "dino_bb_torch": loss_fn(oc, "dino"),
             "refined_search_lib": search, "refined_infonce_lib": infonce}
    for fn in cases.values():   # warm-up of every shape
        fn()
        fn()
    times = {k: [] for k in cases}
    mem = {k: 0.0 for k in cases}
    clock = []
    for _ in range(args.repeats):
        for k, fn in cases.items():   # alternating
            ms, mb = timed(fn, dev)
            times[k].append(ms)
            mem[k] = max(mem[k], mb)
        clock.append(gpu_info())
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    res = {"gpu": gpu_info(), "gpu_samples": clock, "shape": {"H": H, "W": W, "C": C, "frames": N, "pairs": 4, "points": 256},
           "median_ms": med, "peak_extra_MiB": mem, "repeats": args.repeats,
           "tf32_matmul": torch.backends.cuda.matmul.allow_tf32, "time": time.strftime("%Y-%m-%d %H:%M:%S")}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
