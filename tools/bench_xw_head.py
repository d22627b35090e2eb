"""The anchor phase's exact-window head (xw_head: exact arg-max, 15 x 15 window, refiner, softmax sums and certificate of
every map the plan sends down the exact-window path) inside steady-state BASELINE config 2 steps.  GPU only.

  python tools/bench_xw_head.py [--steps 20] [--windows 5] [--head sharp] [--trace DIR] [--split] [--dump DIR]

Inputs: bench.py's config 2 (854 x 476 video, T = 50, C = 1024, 256 query points, seeded features and queries), the
anchor phase forced onto the exact-window pipeline.  Prints one JSON line:
  ms_per_step          the xw_head class per step: CUDA events around each of its launches (the library's profiling
                       brackets), summed over a window of `--steps` infer calls; median over the windows, with min and max
  step_ms              the whole infer step over the same windows (events around the window, brackets on)
  ns_per_map           ms_per_step over the maps of the step that take the exact-window path
  fma_gflops, floor_ms the windowed refiner's 41,760 FMA per map over ms_per_step, and the time those FMAs take at
                       SMs x 128 FMA per clock at the sampled SM clock (the fp32 FMA floor of the class)
  kernels_ms_per_step  torch.profiler, in a run of its own: device time per step of every kernel whose name starts with
                       xw_ (the split of the head class between its kernels, and its neighbours)
  stats                infer_stats() of the last step: exact-window / full-map maps, certificate failures
  gpu                  card name, power limit and the SM clock (NVML, sampled during the timed windows)
  split                with --split: the same timing with the head reduced to its window part (exact arg-max, the
                       15 x 15 window, m_out; dinotrk_xw_head_set_window_only), and the whole head minus it: the time
                       the refiner, softmax sums and certificate add.  (The window-only steps write no track points.)
--dump DIR writes the `anchors` tensor of infer_all for the sharp and the well head (anchors_<head>.npy) and prints their
sha256, so that two builds can be compared byte for byte.
"""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
from bench_coarse import card_info  # noqa: E402

FMA_PER_MAP = 41760   # 169 * 16 * 9 + 121 * 16 * 9


def make_tracker(head, dev, _lib, lib):
    from dino_tracker_b200 import ModelInference, Tracker
    T, C = 50, 1024
    feats = bench.synth_video_features(T, C, dev, 1234, 0.25)
    video = torch.zeros(T, 3, bench.H, bench.W, device=dev)
    model = Tracker(video=video, dino_embed_video=feats, device=dev, delta_channels=[3, 4, 4, 4, C], corr_precision="fp16x3")
    del feats
    model.tracker_head.load_state_dict(bench.head_weights_for(head))
    _lib.check(lib.dinotrk_infer_set_path(1), "infer_set_path")
    return ModelInference(model, model.range_normalizer, 0.7, 0.6)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="infer calls per timed window")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--head", default="sharp", choices=["sharp", "well", "mixed"])
    ap.add_argument("--trace", default=None, metavar="DIR", help="also write the torch.profiler trace there")
    ap.add_argument("--split", action="store_true", help="also time the head's window part alone")
    ap.add_argument("--dump", default=None, metavar="DIR", help="write infer_all's anchors for the sharp and well heads")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_xw_head.py needs a CUDA device"
    dev = "cuda:0"
    torch.cuda.set_device(0)
    import __graft_entry__ as ge
    ge.build()
    from dino_tracker_b200 import _lib
    from dino_tracker_b200 import model_inference as _mi_mod
    lib = _lib.load()
    _mi_mod.DEFAULT_CHUNK_MAPS = 32768
    q = bench.query_lattice(256, 0).to(dev)

    out = {"kernel": "xw_head", "head": a.head}
    if a.dump:
        os.makedirs(a.dump, exist_ok=True)
        digests = {}
        for head in ("sharp", "well"):
            mi = make_tracker(head, dev, _lib, lib)
            anchors = mi.infer_all(q)["anchors"].cpu().numpy()
            np.save(os.path.join(a.dump, f"anchors_{head}.npy"), anchors)
            digests[head] = hashlib.sha256(anchors.tobytes()).hexdigest()
            del mi
            torch.cuda.empty_cache()
        out["anchors_sha256"] = digests

    mi = make_tracker(a.head, dev, _lib, lib)
    for _ in range(a.warmup):
        mi.infer(q)
    torch.cuda.synchronize()
    stats = _lib.infer_stats()

    gpu = card_info()
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.1)
    t0 = time.perf_counter()

    def timed():
        head_ms, step_ms = [], []
        _lib.profile_enable(True)
        for _ in range(a.windows):
            _lib.profile_collect()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                mi.infer(q)
            e1.record()
            torch.cuda.synchronize()
            prof = _lib.profile_collect()
            head_ms.append(prof["xw_head"][0] / a.steps)
            step_ms.append(e0.elapsed_time(e1) / a.steps)
        _lib.profile_enable(False)
        return head_ms, step_ms

    head_ms, step_ms = timed()
    split = None
    if a.split:
        _lib.check(lib.dinotrk_xw_head_set_window_only(1), "xw_head_set_window_only")
        try:
            mi.infer(q)
            torch.cuda.synchronize()
            win_ms, _ = timed()
        finally:
            _lib.check(lib.dinotrk_xw_head_set_window_only(0), "xw_head_set_window_only")
        wm, hm = sorted(win_ms)[len(win_ms) // 2], sorted(head_ms)[len(head_ms) // 2]
        split = {"window_ms_per_step": wm, "window_ms_min": min(win_ms), "window_ms_max": max(win_ms),
                 "refine_and_tail_ms_per_step": hm - wm}
    t1 = time.perf_counter()
    clocks = sampler.stop(t0, t1)

    # per-kernel split, profiler on, in a run of its own
    from torch.profiler import ProfilerActivity, profile
    prof_steps = 5
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(prof_steps):
            mi.infer(q)
        torch.cuda.synchronize()
    kernels = {}
    for ev in p.key_averages():
        if ev.key.startswith("xw_") or "xw_" in ev.key.split("<")[0]:
            dt = getattr(ev, "device_time_total", None)
            if dt is None:
                dt = ev.cuda_time_total
            kernels[ev.key.split("(")[0]] = round(dt / 1e3 / prof_steps, 4)
    if a.trace:
        os.makedirs(a.trace, exist_ok=True)
        p.export_chrome_trace(os.path.join(a.trace, "xw_head_trace.json"))

    med = sorted(head_ms)[len(head_ms) // 2]
    mhz = clocks["sm_mhz"]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    maps = stats["exact_window"]
    floor_ms = FMA_PER_MAP * maps / (sms * 128 * mhz * 1e6) * 1e3 if mhz else None
    out.update({
        "ms_per_step": med, "ms_per_step_min": min(head_ms), "ms_per_step_max": max(head_ms),
        "step_ms": sorted(step_ms)[len(step_ms) // 2], "step_ms_min": min(step_ms), "step_ms_max": max(step_ms),
        "ns_per_map": med * 1e6 / max(maps, 1),
        "fma_gflops": FMA_PER_MAP * maps / (med / 1e3) / 1e9,
        "floor_ms": floor_ms, "floor_frac": (floor_ms / med) if floor_ms else None,
        "kernels_ms_per_step": kernels, "split": split, "stats": stats, "steps_per_window": a.steps, "windows": a.windows,
        "gpu": dict(gpu, sm_mhz=mhz, clock_reasons=clocks["reasons"], clock_samples=clocks["samples"]),
    })
    print(json.dumps(out))


if __name__ == "__main__":
    main()
