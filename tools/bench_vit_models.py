"""DINOv2 feature stage per backbone and facet at 854 x 476, stride 7, two frames per call: device time per frame (CUDA
events, warmed up, median of repeats), the algorithmic rate, and the fp32 oracle (oracle/vit_swiglu_facets.py) on the
same frames on the GPU as the torch comparator.  GPU only; weights are seeded random, generated on the GPU.

    python tools/bench_vit_models.py [--reps 7] [--oracle-reps 2] [--no-oracle]

Cases: ViT-g/14 with all 40 blocks (SwiGLU MLP, tap 39, tokens) and ViT-L/14 at tap 15, tokens against keys.
Algorithmic FLOPs per block over N1 = 8108 tokens: 2 N1 (4 D^2 + MLP) + 4 N1^2 D, with MLP = 3 Hd D (SwiGLU: w12 and
w3) or 8 D^2 (GELU); a facet's tap block adds 2 N1 D^2 only.  One JSON line per case, with the card's name, power
limit and SM clocks read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W = 476, 854
CASES = [("dinov2_vitg14", 39, "tokens"), ("dinov2_vitl14", 15, "tokens"), ("dinov2_vitl14", 15, "keys")]


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), (s.strip() for s in r.stdout.splitlines()[0].split(",")))) if r.returncode == 0 else {}


def random_state_dict(name, layer, gen, dev):
    from oracle import vit_swiglu_facets as ovf
    _, dim, _ = ovf.CONFIGS[name]
    hd = ovf.swiglu_hidden(dim) if name == "dinov2_vitg14" else 0

    def rn(*shape, std=0.02):
        return torch.randn(*shape, device=dev, generator=gen) * std
    sd = {"cls_token": rn(1, 1, dim), "pos_embed": rn(1, 1 + 37 * 37, dim), "patch_embed.proj.weight": rn(dim, 3, 14, 14),
          "patch_embed.proj.bias": rn(dim)}
    for i in range(layer + 1):
        p = f"blocks.{i}."
        sd.update({p + "norm1.weight": 1 + rn(dim), p + "norm1.bias": rn(dim), p + "attn.qkv.weight": rn(3 * dim, dim),
                   p + "attn.qkv.bias": rn(3 * dim), p + "attn.proj.weight": rn(dim, dim), p + "attn.proj.bias": rn(dim),
                   p + "ls1.gamma": 1 + rn(dim), p + "norm2.weight": 1 + rn(dim), p + "norm2.bias": rn(dim),
                   p + "ls2.gamma": 1 + rn(dim)})
        if hd:
            sd.update({p + "mlp.w12.weight": rn(2 * hd, dim), p + "mlp.w12.bias": rn(2 * hd),
                       p + "mlp.w3.weight": rn(dim, hd), p + "mlp.w3.bias": rn(dim)})
        else:
            sd.update({p + "mlp.fc1.weight": rn(4 * dim, dim), p + "mlp.fc1.bias": rn(4 * dim),
                       p + "mlp.fc2.weight": rn(dim, 4 * dim), p + "mlp.fc2.bias": rn(dim)})
    return sd, dim, hd


def flops_per_frame(dim, hd, layer, facet, n1):
    mlp = 3 * hd * dim if hd else 8 * dim * dim
    block = 2 * n1 * (4 * dim * dim + mlp) + 4 * n1 * n1 * dim
    return block * (layer + 1) if facet == "tokens" else block * layer + 2 * n1 * dim * dim


def median_ms(fn, reps, warmup=1):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return statistics.median(times), min(times), max(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--oracle-reps", type=int, default=2)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_vit_models needs a CUDA device"
    import oracle
    from dino_tracker_b200 import _lib
    from dino_tracker_b200.vit import DinoV2Features, CONFIGS
    from oracle import vit_swiglu_facets as ovf
    dev = "cuda:0"
    gpu = card()
    n1 = _lib.make_geom(H, W).h * _lib.make_geom(H, W).w + 1
    for name, layer, facet in CASES:
        g = torch.Generator(device=dev).manual_seed(0)
        sd, dim, hd = random_state_dict(name, layer, g, dev)
        frames = torch.rand(2, 3, H, W, device=dev, generator=g)
        ex = DinoV2Features.from_name(name, sd, layer=layer, device=dev, frames_per_call=2, facet=facet)
        med, lo, hi = median_ms(lambda: ex(frames), a.reps)
        fl = flops_per_frame(dim, hd, layer, facet, n1)
        r = {"model": f"{name}@block{layer}", "facet": facet, "swiglu_hidden": hd, "frames_per_call": 2,
             "ms_per_frame": med / 2, "ms_per_frame_min_max": [lo / 2, hi / 2], "reps": a.reps,
             "tflop_per_frame": fl / 1e12, "tflops": fl / (med / 2 / 1000) / 1e12, "card": gpu}
        del ex
        if not a.no_oracle:
            oracle.use_exact_fp32()
            heads = CONFIGS[name][2]
            with torch.no_grad():
                om, _, _ = median_ms(lambda: ovf.dino_features_video(frames, sd, heads, layer, facet=facet), a.oracle_reps)
            r["oracle_fp32_ms_per_frame"] = om / 2
            r["speedup_vs_oracle"] = om / med
        print(json.dumps(r), flush=True)
        del sd, frames
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
