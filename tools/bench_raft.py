"""RAFT-large flow: the library (dino_tracker_b200.raft.RaftLarge) against torchvision's raft_large in fp32 (TF32 off)
and with TF32 on, the same seeded weights, runs alternated.  Prints one JSON line.

  --pair:    one pair at 480 x 856, 24 updates (the library's time includes encoding both frames);
  --direct:  one start frame's 49 direct pairs, both directions (98 flows; library: 50 frames encoded once).
Executed GFMA per pair are counted from the layer shapes (tools-side arithmetic, not measured)."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import raft as oraft  # noqa: E402


def gfma_per_pair(H, W, n, library, frames_per_pair=2.0):
    """Multiply-adds of one flow counted from the layer shapes.  torchvision: 3 encoder runs (feature encoder on both
    frames, context encoder on the first), n mask + upsampling passes, exact N.  Library (executed): the weight rows
    padded as the GEMM runs them (N = 2 -> 64, 126 -> 128, 192 -> 256, 576 -> 768), one mask pass, and per pair
    ``frames_per_pair`` feature-encoder runs plus one context-encoder run per start frame (2 and 1 for a single pair;
    a video's pairs share them)."""
    h, w = H // 8, W // 8
    hw = h * w
    h2, w2, h4, w4 = H // 2, W // 2, H // 4, W // 4
    pad = (lambda n_: 64 if n_ <= 64 else 128 if n_ <= 128 else -(-n_ // 256) * 256) if library else (lambda n_: n_)
    enc = (h2 * w2 * 64 * 3 * 49 + 4 * h2 * w2 * 64 * 64 * 9 + h4 * w4 * 96 * (64 * 9 + 96 * 9 * 3 + 64)
           + hw * 128 * (96 * 9 + 128 * 9 * 3 + 96) + hw * pad(256) * 128)
    corr = hw * hw * 256
    upd = hw * (324 * 256 + 256 * 9 * pad(192) + 2 * 49 * 128 + 128 * 9 * 64 + 256 * 9 * pad(126)
                + 5 * 384 * (2 * 256 + 2 * 128) + 128 * 9 * 256 + 256 * 9 * pad(2))
    mask = hw * (128 * 9 * 256 + 256 * pad(576)) + H * W * 2 * 9
    n_enc = 3 if not library else frames_per_pair + 1
    return (n_enc * enc + corr + n * upd + (n if not library else 1) * mask) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--H", type=int, default=480)
    ap.add_argument("--W", type=int, default=856)
    ap.add_argument("--updates", type=int, default=24)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--direct", type=int, default=49, help="direct pairs of one start frame (0: skip)")
    a = ap.parse_args()
    from dino_tracker_b200.raft import RaftLarge
    dev = "cuda:0"
    model = oraft.seeded_model().to(dev)
    lib = RaftLarge(model, device=dev)
    T = a.direct + 1 if a.direct else 2
    video = torch.cat([oraft.textured_pair(a.H, a.W, (0.5 * t, 0.3 * t))[1] for t in range(T)]).to(dev)

    def tv(x, y, tf32):
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
        return oraft.torchvision_flow(model, x, y, a.updates)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    runs = {"pair_lib": lambda: lib(video[:1], video[1:2]),
            "pair_tv_fp32": lambda: tv(video[:1], video[1:2], False),
            "pair_tv_tf32": lambda: tv(video[:1], video[1:2], True)}
    if a.direct:
        src, dst = video[:1].expand(a.direct, -1, -1, -1), video[1:]
        pairs = [(0, t) for t in range(1, T)] + [(t, 0) for t in range(1, T)]
        runs["direct_lib"] = lambda: lib.flows(lib.encode(video), pairs, a.updates)

        def tv_direct(tf32):
            out = []
            for i in range(0, a.direct, 16):
                out.append(tv(src[i:i + 16], dst[i:i + 16], tf32))
                out.append(tv(dst[i:i + 16], src[i:i + 16], tf32))
            return out
        runs["direct_tv_fp32"] = lambda: tv_direct(False)
        runs["direct_tv_tf32"] = lambda: tv_direct(True)
    times = {k: [] for k in runs}
    peak = {}
    for k, fn in runs.items():   # warm-up of every shape
        fn()
    for _ in range(a.reps):
        for k, fn in runs.items():
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            ms, _ = timed(fn)
            times[k].append(ms)
            peak[k] = max(peak.get(k, 0), torch.cuda.max_memory_allocated() - base)
    gpu = torch.cuda.get_device_name()
    import subprocess
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                               capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    print(json.dumps({"what": "raft_large", "H": a.H, "W": a.W, "updates": a.updates, "gpu": gpu, "power_limit_max_sm": power,
                      "median_ms": {k: round(statistics.median(v), 2) for k, v in times.items()},
                      "all_ms": {k: [round(x, 2) for x in v] for k, v in times.items()},
                      "peak_extra_GiB": {k: round(v / 2**30, 2) for k, v in peak.items()},
                      "gfma_per_pair": {"torchvision": round(gfma_per_pair(a.H, a.W, a.updates, False), 1),
                                        "library_single_pair": round(gfma_per_pair(a.H, a.W, a.updates, True), 1),
                                        "library_direct_98": round(gfma_per_pair(a.H, a.W, a.updates, True, T / 98), 1)}}))


if __name__ == "__main__":
    main()
