"""The anchor phase's exact box GEMM (xw_exact_gemm: split-precision contraction of each cell's descriptors with its 21 x 21
token box) on its own, at the shapes one steady-state chunk of BASELINE config 2 gives it.  GPU only.

  python tools/bench_xw_gemm.py [--launches 1000] [--windows 5]

Inputs: seeded features of the chunk's three anchor frames (P = 67 x 121 = 8107 tokens, C = 1024, split into fp16 hi / lo,
and the same split interleaved per 32 channels);
655 cells of T = 50 maps (32,750 descriptor rows), as in the first full anchor chunk of config 2 (tools/bench_coarse.py):
175 cells anchored in frame 0, 256 in frame 1, 224 in frame 2.  Box origins are drawn from a seed, about a quarter of the
boxes hanging over the border of the token grid (zero-filled there).

Both token-row layouts are timed, alternating window by window: `split` (separate hi / lo halves, 64-byte rows) and
`hilo` (the interleaved split in the feature struct, 128-byte rows).  Prints one JSON line; per layout:
  ms_per_launch        CUDA events around dinotrk_xw_box_gemm, median over the windows, with min and max
  useful_tflops        2 * maps * 441 * C * 3 (three split-precision products per box token) over ms_per_launch
  executed_tflops      the MMA work the kernel issues: per cell of T <= 64 maps, 64 descriptor rows x 448 box columns
                       (m64n256 + m64n192) x C x 3
  clocks_per_64ch      ms_per_launch x SM clock x CTAs / (cells x C / 64): the period of 64 channels of one cell on one
                       SM, epilogue included (2,688 clocks of MMA at the full fp16 rate of 2,048 FMA per clock per SM)
  clocks_per_stage     the same per 32-channel ring stage (1,344 clocks of MMA)
  xbox_sha256          digest of the accumulators, to compare builds and layouts bit for bit
and once:
  gpu                  card name, power limit and the SM clock (NVML, sampled during the timed windows)
"""
import argparse
import ctypes
import hashlib
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from bench_coarse import card_info, time_windows  # noqa: E402  (tools/ is on sys.path when run as a script)

T, GH, GW, C = 50, bench.GEO_H, bench.GEO_W, 1024
P = GH * GW
CELLS = ((0, 175), (1, 256), (2, 224))   # (anchor frame, cells of T maps)
BOX, COLS = 21, 448
EXEC_ROWS, EXEC_COLS = 64, 448            # MMA tile per cell of T <= 64 maps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=1000, help="launches per timed window (>= 20)")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    assert a.launches >= 20
    assert torch.cuda.is_available(), "bench_xw_gemm.py needs a CUDA device"
    dev = "cuda:0"
    torch.cuda.set_device(0)
    import __graft_entry__ as ge
    ge.build()
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    st = _lib.stream_ptr()

    g = torch.Generator(device=dev).manual_seed(2025)
    n_frames = len(CELLS)
    feats = torch.randn(n_frames, P, C, device=dev, generator=g)
    norms = feats.norm(dim=2).contiguous()
    f_hi, f_lo = _lib.split_fp16(feats, st)
    layouts = {"split": _lib.make_features(feats, norms, f_hi, f_lo),
               "hilo": _lib.make_features(feats, norms, f_hi, f_lo, hilo=_lib.split_hilo(feats, st))}
    n_cells = sum(n for _, n in CELLS)
    rows = n_cells * T
    desc = torch.randn(rows, C, device=dev, generator=g)
    d_hi, d_lo = _lib.split_fp16(desc, st)
    del desc
    frame = torch.tensor(np.repeat([f for f, _ in CELLS], [n for _, n in CELLS]), dtype=torch.int32, device=dev)
    m = torch.full((n_cells,), T, dtype=torch.int32, device=dev)
    row0 = torch.arange(n_cells, dtype=torch.int32, device=dev) * T
    rng = np.random.default_rng(7)
    org = np.stack([rng.integers(-6, GH - BOX + 7, n_cells), rng.integers(-6, GW - BOX + 7, n_cells)], 1).astype(np.int32)
    border = int(((org[:, 0] < 0) | (org[:, 0] > GH - BOX) | (org[:, 1] < 0) | (org[:, 1] > GW - BOX)).sum())
    org_d = torch.from_numpy(org).to(dev).contiguous()
    geom = _lib.make_geom(14 + 7 * (GH - 1), 14 + 7 * (GW - 1))
    xbox = torch.zeros(rows, COLS, dtype=torch.float32, device=dev)

    def gemm_of(fs):
        args = (ctypes.byref(fs), ctypes.byref(geom), _lib.ptr(d_hi), _lib.ptr(d_lo), rows, _lib.ptr(row0), _lib.ptr(m),
                _lib.ptr(frame), _lib.ptr(org_d), n_cells, T, _lib.ptr(xbox), st)
        return lambda: _lib.check(lib.dinotrk_xw_box_gemm(*args), "xw_box_gemm")

    gemms = {name: gemm_of(fs) for name, fs in layouts.items()}
    digest = {}
    for name, gemm in gemms.items():
        xbox.zero_()
        for _ in range(a.warmup):
            gemm()
        torch.cuda.synchronize()
        digest[name] = hashlib.sha256(xbox[:, :BOX * BOX].cpu().numpy().tobytes()).hexdigest()

    gpu = card_info()
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.1)
    t0 = time.perf_counter()
    call_ms = {name: [] for name in gemms}
    for _ in range(a.windows):   # the layouts alternate window by window
        for name, gemm in gemms.items():
            call_ms[name] += time_windows(gemm, a.launches, 1)
    t1 = time.perf_counter()
    clocks = sampler.stop(t0, t1)

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = min(n_cells, sms)
    mhz = clocks["sm_mhz"]
    useful = 2.0 * rows * BOX * BOX * C * 3
    executed = 2.0 * n_cells * EXEC_ROWS * EXEC_COLS * C * 3
    legs = {}
    for name, ms in call_ms.items():
        med = sorted(ms)[len(ms) // 2]
        sec = med / 1e3
        legs[name] = {
            "ms_per_launch": med, "ms_per_launch_min": min(ms), "ms_per_launch_max": max(ms),
            "useful_tflops": useful / sec / 1e12, "executed_tflops": executed / sec / 1e12,
            "clocks_per_64ch": (sec * mhz * 1e6 * ctas / (n_cells * C / 64)) if mhz else None,
            "clocks_per_stage": (sec * mhz * 1e6 * ctas / (n_cells * -(-C // 32))) if mhz else None,
            "xbox_sha256": digest[name],
        }
    print(json.dumps({
        "kernel": "xw_exact_gemm (xw_gemm_kernel<64, HILO>)",
        "shape": {"T": T, "P": P, "C": C, "cells": n_cells, "rows": rows, "boxes_over_the_border": border, "ctas": ctas},
        "launches_per_window": a.launches, "windows": a.windows,
        "layouts": legs, "same_xbox": digest["split"] == digest["hilo"],
        "gpu": dict(gpu, sm_mhz=mhz, clock_reasons=clocks["reasons"], clock_samples=clocks["samples"]),
    }))


if __name__ == "__main__":
    main()
