"""Delta-DINO's training forward + backward on one chunk of frames, three ways, and the whole training step with each
delta-DINO path (CUDA events, warm-up, alternating repeats; FLOP counts from the shapes; card name, power limit and SM
clock read in the same run).  Prints one JSON object.

    python tools/bench_delta_train.py [--B 4] [--H 476] [--W 854] [--reps 5]

Ways: ``node`` = train.DeltaTrainFunction (split-precision wgmma convolutions), ``graph_fp32`` / ``graph_tf32`` =
``DeltaDINO.forward_graph`` with cuDNN's TF32 off / on.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

SHIPPED = [3, 64, 128, 256, 1024]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q}


def conv_flops(B, H, W, chans):
    """(forward, weight-gradient, input-gradient) FLOPs of the four convolutions (2 per multiply-add)."""
    fwd = dgrad = 0
    h, w = H, W
    for l in range(4):
        f = 2 * B * h * w * chans[l + 1] * 25 * chans[l]
        fwd += f
        if l:
            dgrad += f
        if l < 3:
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    return fwd, fwd, dgrad


def timed(fn):
    e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    e[0].record()
    fn()
    e[1].record()
    torch.cuda.synchronize()
    return e[0].elapsed_time(e[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=4)
    ap.add_argument("--H", type=int, default=476)
    ap.add_argument("--W", type=int, default=854)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--points", type=int, default=512)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from dino_tracker_b200 import Tracker, _lib
    from dino_tracker_b200.networks import DeltaDINO
    from oracle import delta_dino as od
    from oracle import synth
    dev = "cuda:0"
    B, H, W = args.B, args.H, args.W
    h, w = 1 + (H - 14) // 7, 1 + (W - 14) // 7
    sd = od.random_state_dict(SHIPPED, torch.Generator().manual_seed(1), last_std=0.01)
    m = DeltaDINO(channels=SHIPPED, vit_stride=7).to(dev)
    m.load_state_dict(sd)
    m.train()
    frames = synth.random_video(B, H, W, seed=2).to(dev)
    gr = torch.randn(B, SHIPPED[-1], h, w, generator=torch.Generator().manual_seed(3)).to(dev) * 1e-7
    dummy = torch.empty(B, SHIPPED[-1], h, w, device=dev)

    def node():
        (m(frames, dummy) * gr).sum().backward()

    def graph(tf32):
        def run():
            torch.backends.cudnn.allow_tf32 = tf32
            (m.forward_graph(frames, (h, w)) * gr).sum().backward()
        return run

    ways = {"node": node, "graph_fp32": graph(False), "graph_tf32": graph(True)}
    for fn in ways.values():
        for _ in range(args.warmup):
            fn()
    ms = {k: [] for k in ways}
    for _ in range(args.reps):
        for k, fn in ways.items():
            m.zero_grad(set_to_none=True)
            ms[k].append(timed(fn))
    torch.backends.cudnn.allow_tf32 = False
    _lib.profile_enable(True)
    _lib.profile_collect()
    node()
    torch.cuda.synchronize()
    prof = {k: round(v[0], 3) for k, v in _lib.profile_collect().items()}
    _lib.profile_enable(False)
    f_fwd, f_wg, f_dg = conv_flops(B, H, W, SHIPPED)
    chunk = {k: {"median_ms": statistics.median(v), "min_ms": min(v), "ms": [round(x, 3) for x in v],
                 "conv_tflops_per_s": (f_fwd + f_wg + f_dg) / (statistics.median(v) * 1e-3) / 1e12} for k, v in ms.items()}

    # the whole training step: model(inputs) + Huber + norm regulariser + backward, per delta-DINO path
    T, C = B, SHIPPED[-1]
    feats = synth.random_features(T, C, h, w, seed=4)
    feats = feats / feats.norm(dim=1, keepdim=True)
    tr = Tracker(video=frames, dino_embed_video=feats, device=dev, delta_channels=SHIPPED)
    tr.tracker_head.load_state_dict(synth.head_weights("well", seed=5))
    tr.delta_dino.load_state_dict(sd)
    tr.train()
    g = torch.Generator().manual_seed(6)
    P = args.points
    pts = (torch.rand(P, 3, generator=g) * torch.tensor([W - 1.0, H - 1.0, 0.0])).to(dev)
    inp = (pts, torch.randint(0, T, (P,), generator=g).to(dev), torch.randint(0, T, (P,), generator=g).to(dev),
           torch.arange(T, dtype=torch.int32, device=dev))
    labels = (torch.rand(P, 2, generator=g) * 2 - 1).to(dev)
    huber = torch.nn.HuberLoss(delta=1 / 32)

    def step(precision, tf32):
        def run():
            # conv_precision selects the delta-DINO path of a forward with a graph: "fp16x3" = the node, "fp32" = forward_graph
            tr.delta_dino.conv_precision = precision
            torch.backends.cudnn.allow_tf32 = tf32
            c = tr(inp)
            reg = (tr.frame_embeddings.norm(dim=1) / tr.raw_embeddings.norm(dim=1) - 1).abs().mean()
            (huber(c, labels) + 1e-4 * reg).backward()
        return run

    steps = {"node": step("fp16x3", False), "graph_fp32": step("fp32", False), "graph_tf32": step("fp32", True)}
    for fn in steps.values():
        for _ in range(args.warmup):
            fn()
    sms = {k: [] for k in steps}
    for _ in range(args.reps):
        for k, fn in steps.items():
            tr.zero_grad(set_to_none=True)
            sms[k].append(timed(fn))
    tr.delta_dino.conv_precision = "fp16x3"
    torch.backends.cudnn.allow_tf32 = False
    out = {"card": card(), "shape": {"B": B, "H": H, "W": W, "widths": SHIPPED, "points": P},
           "flop": {"forward": f_fwd, "weight_grad": f_wg, "input_grad": f_dg},
           "chunk_forward_backward": chunk, "node_kernel_ms": prof,
           "training_step": {k: {"median_ms": statistics.median(v), "ms": [round(x, 3) for x in v]} for k, v in sms.items()}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
