"""DINO v1 backbones and the int8 coarse pass at ViT-g/14's width.  GPU only; weights and features are seeded random.

    python tools/bench_backbones.py [--reps 7]

1. ViT-S/8 and ViT-B/8 (all 12 blocks, tokens of the last block) on 854 x 476 frames at stride 7 (67 x 121 tokens), two
   frames per call: device time per frame (CUDA events, warmed up, median of repeats) and the algorithmic rate
   (tools/bench_vit_models.py's FLOP count: 2 N1 (4 D^2 + 8 D^2) + 4 N1^2 D per block, N1 = 8108).
2. xw_coarse_gemm at C = 1536 on one config-2-shaped chunk (tools/bench_coarse.py --C 1536, run as a subprocess): the
   fp16 pass and the int8 pass, ms per launch and their ratio.
Every JSON line carries the card's name and power limit, and the SM clock sampled (NVML) during its own timed windows."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

H, W = 476, 854


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_backbones needs a CUDA device"
    import bench
    import bench_vit_models as bvm
    from dino_tracker_b200 import _lib
    from dino_tracker_b200.vit import DinoV2Features
    from oracle import vit_dino_v1 as ov1
    dev = "cuda:0"
    geom = _lib.make_geom(H, W, 8, 7, 35)
    n1 = geom.h * geom.w + 1
    for name, (depth, dim, heads) in ov1.CONFIGS.items():
        g = torch.Generator(device=dev).manual_seed(0)
        sd = {k: v.to(dev) for k, v in ov1.random_state_dict(depth, dim, torch.Generator().manual_seed(0)).items()}
        frames = torch.rand(2, 3, H, W, device=dev, generator=g)
        ex = DinoV2Features.from_name(name, sd, device=dev, frames_per_call=2)
        ex(frames)
        torch.cuda.synchronize()
        sampler = bench.ClockSampler(0)
        sampler.start()
        time.sleep(0.1)
        t0 = time.perf_counter()
        med, lo, hi = bvm.median_ms(lambda: ex(frames), a.reps)
        clocks = sampler.stop(t0, time.perf_counter())
        fl = bvm.flops_per_frame(dim, 0, depth - 1, "tokens", n1)
        print(json.dumps({"model": name, "blocks": depth, "facet": "tokens", "grid": [geom.h, geom.w], "frames_per_call": 2,
                          "ms_per_frame": med / 2, "ms_per_frame_min_max": [lo / 2, hi / 2], "reps": a.reps,
                          "tflop_per_frame": fl / 1e12, "tflops": fl / (med / 2 / 1000) / 1e12, "card": bvm.card(),
                          "sm_mhz_sampled": clocks["sm_mhz"], "clock_reasons": clocks["reasons"],
                          "clock_samples": clocks["samples"]}),
              flush=True)
        del ex, sd, frames
        torch.cuda.empty_cache()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_coarse.py"), "--C", "1536"], check=True,
                       stdout=subprocess.PIPE, text=True)
    c = json.loads(r.stdout.strip().splitlines()[-1])
    print(json.dumps({"kernel": "xw_coarse_gemm", "C": 1536, "shape": c["shape"], "fp16_ms_per_launch": c["ms_per_launch"],
                      "fp16_ms_min_max": [c["ms_per_launch_min"], c["ms_per_launch_max"]],
                      "int8_ms_per_launch": c["int8"]["ms_per_launch"],
                      "int8_ms_min_max": [c["int8"]["ms_min"], c["int8"]["ms_max"]],
                      "fp16_over_int8": c["int8"]["speedup_vs_fp16"], "int8_eps_max": c["int8"]["eps_max"],
                      "gpu": c["gpu"], "int8_sm_mhz": c["int8"]["gpu"]["sm_mhz"], "card": bvm.card()}), flush=True)


if __name__ == "__main__":
    main()
