"""Time the best-buddy preprocessing kernels against the oracle's torch path (the reference's arithmetic) on one GPU.

    python tools/bench_preprocess.py [--frames 50 100] [--reps 3] [--out results/bench_preprocess.json]

Per video length T at 476 x 854 (the project's video size): seeded smooth flows (precomputed on the GPU; RAFT is not
timed) and a best-buddy dict from the library's kernel on seeded C = 64 features.  It times
  - chaining without direct flow (``chain_trajectories``) and the oracle's restatement of extract_trajectories.py;
  - chaining with direct flow (direct flows produced on the fly by a cheap difference of fields in both paths);
  - the flow filter (``of_filter``) and the oracle's restatement of of_filter_dino_best_buddies.py;
and reports M, a digest of both outputs (equal digests = identical outputs), and the card's name and power limit read
in the same process.  The oracle runs once per T (it takes seconds to minutes); the library path takes the median of
``--reps`` runs after one warm-up.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def fields(T, H, W, seed, dev):
    """Smooth motion field per frame (low-frequency cosines, 3 px amplitude); flow(a, b) = field[b] - field[a]."""
    g = torch.Generator().manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32), torch.arange(W, device=dev, dtype=torch.float32),
                            indexing="ij")
    out = torch.zeros(T, 2, H, W, device=dev)
    for t in range(T):
        for c in range(2):
            for _ in range(3):
                a, fx, fy, ph = torch.rand(4, generator=g).tolist()
                out[t, c] += 3.0 * (a - 0.5) * torch.cos(2 * torch.pi * (fx * xs / W * 2 + fy * ys / H * 2) + 6.3 * ph)
    return out


def digest(x):
    return hashlib.sha256(x.detach().float().nan_to_num(-12345.0).cpu().numpy().tobytes()).hexdigest()[:16]


def bb_digest(d):
    h = hashlib.sha256()
    for k in d:
        for f in ("source_coords", "target_coords", "cos_sims"):
            v = d[k][f]
            h.update(b"none" if v is None else v.float().cpu().numpy().tobytes())
    return h.hexdigest()[:16]


def timed(fn, reps):
    ts, out = [], None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2] * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[50, 100])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_preprocess needs a CUDA device")
    from dino_tracker_b200.best_buddies import best_buddies, of_filter
    from dino_tracker_b200.trajectories import chain_trajectories
    from oracle import of_filter as oof
    from oracle import synth
    from oracle import trajectories as otr
    from oracle.tracker import Geometry
    dev = torch.device("cuda:0")
    H, W, thr, dthr = 476, 854, 1.0, 2.0
    res = {"card": card(), "H": H, "W": W, "runs": []}
    for T in args.frames:
        F = fields(T, H, W, seed=T, dev=dev)
        fwd, bwd = (F[1:] - F[:-1]).contiguous(), (F[:-1] - F[1:]).contiguous()

        def direct(s):
            return (F[s + 1:] - F[s:s + 1]).contiguous(), (F[s:s + 1] - F[s + 1:]).contiguous()
        geo = Geometry(H=H, W=W)
        feats, _ = synth.shifted_field_features(T, 64, geo.h, geo.w, seed=T, noise=0.5, max_shift=2)
        bb = best_buddies(feats, H, W)
        del feats
        run = {"T": T, "bb_pairs_kept": sum(int(v["source_coords"].shape[0]) for v in bb.values())}
        chain_trajectories(fwd, bwd, None, thr, 2)                      # warm-up
        run["chain_ms"], traj = timed(lambda: chain_trajectories(fwd, bwd, None, thr, 2), args.reps)
        run["chain_direct_ms"], traj_d = timed(lambda: chain_trajectories(fwd, bwd, direct, thr, 2, dthr), args.reps)
        of_filter(bb, traj, H, W, 7)
        run["of_filter_ms"], filt = timed(lambda: of_filter(bb, traj, H, W, 7), args.reps)
        run.update(M=int(traj.shape[0]), M_direct=int(traj_d.shape[0]), chain_digest=digest(traj),
                   chain_direct_digest=digest(traj_d), of_filter_digest=bb_digest(filt))
        if not args.no_oracle:
            run["oracle_chain_ms"], o = timed(lambda: otr.extract_trajectories(fwd, bwd, None, thr, 2), 1)
            run.update(oracle_M=int(o.shape[0]), oracle_chain_digest=digest(o))
            del o
            run["oracle_chain_direct_ms"], o = timed(lambda: otr.extract_trajectories(fwd, bwd, direct, thr, 2, dthr), 1)
            run.update(oracle_M_direct=int(o.shape[0]), oracle_chain_direct_digest=digest(o))
            del o
            run["oracle_of_filter_ms"], o = timed(lambda: oof.of_filter(bb, traj, H, W, 7), 1)
            run["oracle_of_filter_digest"] = bb_digest(o)
        res["runs"].append(run)
        print(json.dumps(run), flush=True)
        del traj, traj_d, filt, bb, F, fwd, bwd
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
