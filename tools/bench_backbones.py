"""DINO v1 backbones and the int8 coarse pass at ViT-g/14's width.  GPU only; weights and features are seeded random.

    python tools/bench_backbones.py [--reps 7] [--only {all,v1,dinov3}]

1. ViT-S/8 and ViT-B/8 (all 12 blocks, tokens of the last block) on 854 x 476 frames at stride 7 (67 x 121 tokens), two
   frames per call: device time per frame (CUDA events, warmed up, median of repeats) and the algorithmic rate
   (tools/bench_vit_models.py's FLOP count: 2 N1 (4 D^2 + 8 D^2) + 4 N1^2 D per block, N1 = 8108).
2. xw_coarse_gemm at C = 1536 on one config-2-shaped chunk (tools/bench_coarse.py --C 1536, run as a subprocess): the
   fp16 pass and the int8 pass, ms per launch and their ratio.
3. DINOv3 ViT-L/16 (all 24 blocks, 4 registers) on 854 x 476 frames at stride 8 (58 x 105 tokens, N1 = 6095) and 16
   (29 x 53, N1 = 1542), alternated call by call with DINOv2 ViT-L/14 at stride 7 (N1 = 8108), two frames per call: ms per
   frame and the algorithmic rate with the same FLOP count.  Then the qkv stage at D = 1024 on two stride-8 frames with
   and without the rotary epilogue (dinotrk_vit_stage_ext, CUDA events over 20 launches, alternated, median of repeats).
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


def _timed(fn, n=1):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def _stats(ts):
    import statistics
    return statistics.median(ts), min(ts), max(ts)


def dinov3(reps):
    import bench
    import bench_vit_models as bvm
    import ctypes
    from dino_tracker_b200 import _lib
    from dino_tracker_b200.vit import DinoV2Features, DinoV3Features, rope_table
    from oracle import vit_dinov3 as ov3
    dev = "cuda:0"
    frames = torch.rand(2, 3, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    v2 = DinoV2Features.from_name("dinov2_vitl14", bvm.random_state_dict("dinov2_vitl14", 23, torch.Generator(device=dev).manual_seed(0), dev)[0],
                                  device=dev, frames_per_call=2)
    sd3 = {k: v.to(dev) for k, v in ov3.random_state_dict(24, 1024, torch.Generator().manual_seed(0)).items()}
    runs = {"dinov2_vitl14 s7": (v2, 7, 1), "dinov3_vitl16 s8": (DinoV3Features(sd3, stride=8, device=dev, frames_per_call=2), 8, 5),
            "dinov3_vitl16 s16": (DinoV3Features(sd3, stride=16, device=dev, frames_per_call=2), 16, 5)}
    for ex, _, _ in runs.values():
        ex(frames)
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.1)
    t0 = time.perf_counter()
    for _ in range(reps):
        for k, (ex, _, _) in runs.items():
            times[k].append(_timed(lambda: ex(frames)))
    clocks = sampler.stop(t0, time.perf_counter())
    for k, (ex, stride, pre) in runs.items():
        geom = _lib.make_geom(H, W, ex.patch, stride, 35)
        n1 = geom.h * geom.w + pre
        med, lo, hi = _stats(times[k])
        fl = bvm.flops_per_frame(1024, 0, 23, "tokens", n1)
        print(json.dumps({"model": k, "blocks": 24, "grid": [geom.h, geom.w], "N1": n1, "frames_per_call": 2,
                          "ms_per_frame": med / 2, "ms_per_frame_min_max": [lo / 2, hi / 2], "reps": reps,
                          "tflop_per_frame": fl / 1e12, "tflops": fl / (med / 2 / 1000) / 1e12, "card": bvm.card(),
                          "sm_mhz_sampled": clocks["sm_mhz"], "clock_reasons": clocks["reasons"]}), flush=True)
    del runs, v2
    torch.cuda.empty_cache()
    # the qkv stage with and without the rotary epilogue, same shapes
    lib = _lib.load()
    geom = _lib.make_geom(H, W, 16, 8, 35)
    D, B, R = 1024, 2, 4
    rows = B * (geom.h * geom.w + 1 + R)
    g = torch.Generator(device=dev).manual_seed(1)
    y = torch.randn(rows, D, device=dev, generator=g).half()
    w = (torch.randn(3 * D, D, device=dev, generator=g) * D ** -0.5).half()
    bias = torch.randn(3 * D, device=dev, generator=g) * 0.05
    q, k, vT = (torch.empty(B * D * (rows // B + 8), device=dev, dtype=torch.half) for _ in range(3))
    ws = torch.empty(4096, device=dev, dtype=torch.uint8)
    table = rope_table(geom.h, geom.w, 100.0, dev)
    cfg = _lib.VitConfig(1, D, D // 64, 0, 16, 8, 0, 1, 1)
    wts = {}
    for name, tab in (("qkv", None), ("qkv+rope", table)):
        wt = _lib.VitWeights()
        wt.n_registers, wt.rope = R, None if tab is None else tab.data_ptr()
        wts[name] = wt

    def stage(wt):
        _lib.check(lib.dinotrk_vit_stage_ext(2, ctypes.byref(cfg), ctypes.byref(wt), ctypes.byref(geom), B, _lib.ptr(y), _lib.ptr(w),
                                             _lib.ptr(bias), None, _lib.ptr(q), _lib.ptr(k), _lib.ptr(vT), _lib.ptr(ws),
                                             ws.numel(), _lib.stream_ptr()), "vit_stage_ext")
    st = {n: [] for n in wts}
    for n, wt in wts.items():
        _timed(lambda: stage(wt), 5)
    for _ in range(3 * reps):
        for n, wt in wts.items():
            st[n].append(_timed(lambda: stage(wt), 20))
    flop = 2 * rows * 3 * D * D
    med = {n: _stats(t) for n, t in st.items()}
    print(json.dumps({"kernel": "vit qkv stage", "D": D, "rows": rows, "cta_pairs": True,
                      **{f"{n}_ms": m[0] for n, m in med.items()}, **{f"{n}_ms_min_max": [m[1], m[2]] for n, m in med.items()},
                      **{f"{n}_tflops": flop / (m[0] / 1000) / 1e12 for n, m in med.items()},
                      "rope_over_plain": med["qkv+rope"][0] / med["qkv"][0], "card": bvm.card()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--only", choices=["all", "v1", "dinov3"], default="all")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_backbones needs a CUDA device"
    if a.only in ("all", "dinov3"):
        dinov3(a.reps)
    if a.only == "dinov3":
        return
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
