"""Bench-scale A/B of the two correlation-GEMM precisions (wgmma split-fp16, three passes, vs exact-fp32 FFMA):
max trajectory difference, occlusion mismatches, anchor-track differences, timing.  GPU only."""
import argparse
import sys
import os
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from bench_inputs import sharp_head  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=50)
    ap.add_argument("--C", type=int, default=1024)
    ap.add_argument("--nq", type=int, default=256)
    ap.add_argument("--noise", type=float, default=0.25)
    a = ap.parse_args()
    from dino_tracker_b200 import ModelInference, Tracker
    dev = "cuda:0"
    feats = bench.synth_video_features(a.T, a.C, dev, 1234, a.noise)
    video = torch.zeros(a.T, 3, bench.H, bench.W, device=dev)
    q = bench.query_lattice(a.nq, 0).to(dev)
    res = {}
    for prec in ("fp32", "fp16x3"):
        m = Tracker(video=video, dino_embed_video=feats, device=dev, delta_channels=[3, 4, 4, 4, a.C], corr_precision=prec)
        m.tracker_head.load_state_dict(sharp_head(0))
        mi = ModelInference(m, m.range_normalizer, 0.7, 0.6)
        mi.infer(q); torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = mi.infer_all(q); torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        res[prec] = r
        print(f"{prec}: {dt * 1000:.1f} ms per infer ({a.nq / dt:.0f} qp/s)")
        del m, mi
    A, B = res["fp32"], res["fp16x3"]
    dtraj = (A["traj"] - B["traj"]).abs()
    print("max |traj diff| px:", dtraj.max().item(), " #points > 1e-3:", int((dtraj[..., :2].max(-1).values > 1e-3).sum()))
    print("occlusion mismatches:", int((A["occ"] != B["occ"]).sum()), "of", A["occ"].numel())
    vis = A["cos_sims"] >= 0.7
    da = (A["anchors"] - B["anchors"]).abs().max(-1).values  # N x Ta x Ti
    da = da[vis]
    print("anchor tracks: max diff", da.max().item(), " #>1e-3:", int((da > 1e-3).sum()), " #>1px:", int((da > 1).sum()), "of", da.numel())
    print("cos diff max:", (A["cos_sims"] - B["cos_sims"]).abs().max().item())


if __name__ == "__main__":
    main()
