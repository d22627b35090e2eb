"""The anchor phase's coarse pass (xw_coarse_gemm: CTA-pair fp16 wgmma GEMM + tile-key epilogue) on its own, at the
shapes one steady-state chunk of BASELINE config 2 gives it.  GPU only.

  python tools/bench_coarse.py [--launches 100] [--windows 5] [--C 1024]

Inputs: seeded feature video T = 50, P = 67 x 121 = 8107 tokens, C = 1024 (--C: another channel count, a multiple of
16 up to 2048, so that the time per launch can be fitted against the reduction length: the intercept is the cost per tile
that does not scale with K); one anchor-phase chunk of 32,750 descriptor rows.  With 256 queries that anchor in every
frame, every anchor frame holds 256 x 50 = 12,800 work items; the chunk cap of 32,768 maps cut at whole cells (multiples
of T) is 32,750, and the probe chunk (4,050 items) takes the start of frame 0.  So the first full chunk is frame 0's remaining 8,750 rows, all 12,800 of frame 1 and 11,200 of frame 2.

Prints one JSON line:
  ms_per_launch     CUDA events around dinotrk_xw_coarse_keys, median over the windows, with min and max.  Besides the
                    GEMM the call runs two set-up kernels of a few microseconds (reciprocal token norms over T x P
                    floats, the M-tile prefix); the rates below count them as GEMM time
  tflops            2 * rows * P * C over ms_per_launch
  l2_operand_bytes  what the CTAs load through TMA per launch: per pair tile and K block each CTA loads its 128 A rows
                    and half of the 256 B rows (multicast to both), 2 x 128 x 64 fp16 = 32 KiB
  clocks_per_kblock ms_per_launch x SM clock x CTAs / CTA K blocks: the period of one 64-wide K block of one CTA,
                    epilogue included (1,024 clocks of MMA at the full m64n256k16 rate)
  cublas            torch.matmul fp16 on (M, N, K) = (12,800, 8,107, 1,024), the largest group, same timing (what the
                    tensor cores reach on this card under its power limit; it also writes the 207 MB fp16 product)
  gpu               card name, power limit and the SM clock (NVML, sampled during the timed windows)
  keys_sha256       digest of the keys, to compare builds bit for bit
  int8              the same chunk on the int8 pass (dinotrk_xw_coarse_keys_i8 on dinotrk_quantise_s8 operands): ms, tops
                    (2 * rows * P * C over its time), speedup over the fp16 pass, the largest per-map eps, the SM
                    clock sampled during its own timed windows, and clocks_per_mma_block: ms x SM clock x CTAs over the
                    launch's 128 x 128 x 128 MMA blocks (128 descriptor rows of a CTA, 128 tokens, one 128-channel K
                    block; padding rows, tokens and channels included), 512 clocks at the full int8 rate
"""
import argparse
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

T, GH, GW = 50, bench.GEO_H, bench.GEO_W
P = GH * GW
GROUPS = ((0, 8750), (1, 12800), (2, 11200))   # (anchor frame, descriptor rows)
BM_PAIR, BN, BK = 256, 256, 64                  # CTA-pair tile of the coarse GEMM, fp16 K block (tcgemm.cuh)


def card_info():
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        name = pynvml.nvmlDeviceGetName(h)
        return {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0,
                "sm_max_mhz": pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)}
    except Exception:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], stdout=subprocess.PIPE, text=True).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}


def time_windows(fn, launches, windows):
    """ms per launch of each window of `launches` back-to-back calls (CUDA events)."""
    res = []
    for _ in range(windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res.append(e0.elapsed_time(e1) / launches)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=100, help="launches per timed window (>= 20)")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--C", type=int, default=1024, help="feature channels (a multiple of 16, <= 2048)")
    a = ap.parse_args()
    assert a.launches >= 20
    assert a.C > 0 and a.C % 16 == 0 and a.C <= 2048, "--C: a multiple of 16 up to 2048 (the int8 pass's limits)"
    C = a.C
    assert torch.cuda.is_available(), "bench_coarse.py needs a CUDA device"
    dev = "cuda:0"
    torch.cuda.set_device(0)
    import __graft_entry__ as ge
    ge.build()
    from dino_tracker_b200 import _lib
    lib = _lib.load()

    g = torch.Generator(device=dev).manual_seed(2024)
    feats = torch.randn(T, P, C, device=dev, generator=g)
    norms = feats.norm(dim=2).contiguous()
    hi = feats.half().contiguous()
    fs = _lib.make_features(feats, norms, hi, hi)   # (the coarse pass reads the hi halves only)
    rows = sum(m for _, m in GROUPS)
    desc = torch.randn(rows, C, device=dev, generator=g)
    desc_hi, desc_norm = desc.half().contiguous(), desc.norm(dim=1).contiguous()
    del desc
    frame = torch.tensor([f for f, _ in GROUPS], dtype=torch.int32, device=dev)
    m = torch.tensor([n for _, n in GROUPS], dtype=torch.int32, device=dev)
    row0 = torch.cumsum(m, 0, dtype=torch.int32) - m
    geom = _lib.make_geom(14 + 7 * (GH - 1), 14 + 7 * (GW - 1))
    n_tiles = -(-P // 128)
    key1 = torch.empty(rows, n_tiles, dtype=torch.int64, device=dev)
    max2 = torch.empty(rows, n_tiles, dtype=torch.float32, device=dev)
    nb = lib.dinotrk_xw_coarse_keys_workspace_bytes(T, len(GROUPS), ctypes.byref(geom))
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    args = (ctypes.byref(fs), ctypes.byref(geom), _lib.ptr(desc_hi), rows, _lib.ptr(desc_norm), _lib.ptr(frame), _lib.ptr(row0),
            _lib.ptr(m), len(GROUPS), _lib.ptr(key1), _lib.ptr(max2), _lib.ptr(ws), nb, _lib.stream_ptr())

    def coarse():
        _lib.check(lib.dinotrk_xw_coarse_keys(*args), "xw_coarse_keys")

    fq, ffac, _, frho = _lib.quantise_s8(feats, norms, P, _lib.stream_ptr())
    fs8 = _lib.make_features(feats, norms, hi, hi, quant=(fq, ffac, frho))
    desc8 = desc_hi.float()
    dq, dfac, drho, _ = _lib.quantise_s8(desc8, desc8.norm(dim=1).contiguous(), rows, _lib.stream_ptr())
    del desc8
    eps = torch.empty(rows, dtype=torch.float32, device=dev)
    args8 = (ctypes.byref(fs8), ctypes.byref(geom), _lib.ptr(dq), _lib.ptr(dfac), _lib.ptr(drho), rows, _lib.ptr(frame),
             _lib.ptr(row0), _lib.ptr(m), len(GROUPS), _lib.ptr(key1), _lib.ptr(max2), _lib.ptr(eps), _lib.ptr(ws), nb,
             _lib.stream_ptr())

    def coarse8():
        _lib.check(lib.dinotrk_xw_coarse_keys_i8(*args8), "xw_coarse_keys_i8")

    for _ in range(a.warmup):
        coarse()
    torch.cuda.synchronize()
    digest = hashlib.sha256(key1.cpu().numpy().tobytes() + max2.cpu().numpy().tobytes()).hexdigest()

    gpu = card_info()
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.1)
    t0 = time.perf_counter()
    call_ms = time_windows(coarse, a.launches, a.windows)
    t1 = time.perf_counter()
    clocks = sampler.stop(t0, t1)
    for _ in range(a.warmup):
        coarse8()
    torch.cuda.synchronize()
    sampler8 = bench.ClockSampler(0)
    sampler8.start()
    time.sleep(0.1)
    t0 = time.perf_counter()
    s8_ms = time_windows(coarse8, a.launches, a.windows)
    t1 = time.perf_counter()
    clocks8 = sampler8.stop(t0, t1)
    s8_med = sorted(s8_ms)[len(s8_ms) // 2]

    # cuBLAS yardstick on the largest group's shape, computed as the transposed product F @ D^T: both operands K-major
    # like the coarse GEMM's, and every leading dimension a multiple of 8 (an 8107-wide fp16 output row is not 16-byte
    # aligned, which keeps cuBLAS off its tensor-core kernels)
    mm, nn, kk = 12800, P, C
    x = torch.randn(mm, kk, device=dev, generator=g).half()
    w = torch.randn(nn, kk, device=dev, generator=g).half()
    for _ in range(a.warmup):
        torch.matmul(w, x.t())
    torch.cuda.synchronize()
    mm_ms = time_windows(lambda: torch.matmul(w, x.t()), a.launches, a.windows)

    flop = 2.0 * rows * P * C
    # int8: CTA row blocks of 128 x token blocks of 128 x K blocks of 128 channels
    mma_blocks8 = 2 * sum(-(-n // BM_PAIR) for _, n in GROUPS) * -(-P // 128) * -(-C // 128)
    pair_tiles = sum(-(-n // BM_PAIR) for _, n in GROUPS) * -(-P // BN)
    kblocks = 2 * pair_tiles * -(-C // BK)                     # CTA K blocks per launch
    l2_bytes = kblocks * 2 * 128 * BK * 2                      # A (128 rows) + B half (128 rows), fp16
    ctas = 2 * (torch.cuda.get_device_properties(0).multi_processor_count // 2)
    mhz = clocks["sm_mhz"]
    med = sorted(call_ms)[len(call_ms) // 2]
    sec = med / 1e3
    mm_med = sorted(mm_ms)[len(mm_ms) // 2]
    print(json.dumps({
        "kernel": "xw_coarse_gemm (tc_gemm_pair_kernel<F16, CoarseEpi, 256>)",
        "shape": {"T": T, "P": P, "C": C, "rows": rows, "groups": [{"frame": f, "rows": n} for f, n in GROUPS],
                  "pair_tiles": pair_tiles, "ctas": ctas},
        "launches_per_window": a.launches, "windows": a.windows,
        "ms_per_launch": med, "ms_per_launch_min": min(call_ms), "ms_per_launch_max": max(call_ms),
        "tflops": flop / sec / 1e12,
        "l2_operand_bytes": l2_bytes, "l2_operand_tbs": l2_bytes / sec / 1e12,
        "l2_operand_bytes_per_clk_per_sm": (l2_bytes / sec / (mhz * 1e6) / ctas) if mhz else None,
        "clocks_per_kblock": (sec * mhz * 1e6 * ctas / kblocks) if mhz else None,
        "cublas": {"op": "torch.matmul fp16 (8107 x 1024) @ (12800 x 1024)^T, fp16 output", "ms": mm_med, "ms_min": min(mm_ms),
                   "ms_max": max(mm_ms), "tflops": 2.0 * mm * nn * kk / (mm_med / 1e3) / 1e12},
        "gpu": dict(gpu, sm_mhz=mhz, clock_reasons=clocks["reasons"], clock_samples=clocks["samples"]),
        "keys_sha256": digest,
        "int8": {"ms_per_launch": s8_med, "ms_min": min(s8_ms), "ms_max": max(s8_ms), "tops": flop / (s8_med / 1e3) / 1e12,
                 "speedup_vs_fp16": med / s8_med, "eps_max": eps.max().item(), "mma_blocks": mma_blocks8,
                 "clocks_per_mma_block": (s8_med / 1e3 * clocks8["sm_mhz"] * 1e6 * ctas / mma_blocks8)
                 if clocks8["sm_mhz"] else None,
                 "gpu": {"sm_mhz": clocks8["sm_mhz"], "clock_reasons": clocks8["reasons"], "clock_samples": clocks8["samples"]}},
    }))


if __name__ == "__main__":
    main()
