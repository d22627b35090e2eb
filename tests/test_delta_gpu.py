"""GPU parity: Delta-DINO (implicit-GEMM convs + BlurPool + align + residual add) against the reference
vectors in tests/golden and the oracle."""
import os

import numpy as np
import pytest
import torch

from oracle import delta_dino as od
from oracle import synth
from oracle.tracker import Geometry

from golden_util import GOLDEN_DIR

gpu = pytest.mark.gpu
DEV = "cuda:0"


def load_case(name):
    g = dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))
    H, W, T = (int(v) for v in g["HWT"])
    channels = [int(c) for c in g["channels"]]
    seed = int(g["seed"])
    sd = {k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("sd.")}
    video = synth.random_video(T, H, W, seed=seed)
    geo = Geometry(H=H, W=W)
    dino = synth.random_features(T, channels[-1], geo.h, geo.w, seed=seed + 1)
    return g, geo, channels, sd, video, dino


@gpu
@pytest.mark.parametrize("name", ["delta_small", "delta_full_geom"])
def test_refined_features_match_reference_vectors(name):
    from dino_tracker_b200 import Tracker
    g, geo, channels, sd, video, dino = load_case(name)
    model = Tracker(video=video.to(DEV), dino_embed_video=dino, device=DEV, delta_channels=channels)
    model.delta_dino.load_state_dict(sd)
    model.cache_refined_embeddings()
    refined = model.refined_features.cpu().numpy()
    if "refined" in g:
        assert np.abs(refined - g["refined"]).max() <= 5e-5
    else:
        assert np.abs(refined.reshape(-1)[g["refined_idx"]] - g["refined_vals"]).max() <= 5e-5
    # norms cached with the features
    ref_norm = torch.from_numpy(refined).norm(dim=1).reshape(refined.shape[0], -1)
    assert torch.allclose(model._refined_norms.cpu(), ref_norm, rtol=1e-5)
    # DeltaDINO.forward returns the aligned residual (models/networks/delta_dino.py:53-61)
    with torch.no_grad():                        # the CUDA kernels (folded eval-mode BatchNorm)
        res = model.delta_dino(video[:1].to(DEV), dino[:1].to(DEV)).cpu()
    ref_res = od.align_cnn_to_vit(od.delta_cnn(video[:1], sd), (geo.h, geo.w))
    assert (res - ref_res).abs().max().item() <= 5e-5
    # with gradients enabled the same call is a torch graph (training step); in eval mode it is the same function
    import oracle
    oracle.use_exact_fp32()                      # torch's default lets cuDNN convolutions run in TF32
    model.eval()
    res_graph = model.delta_dino(video[:1].to(DEV), dino[:1].to(DEV))
    assert res_graph.requires_grad and (res_graph.detach().cpu() - ref_res).abs().max().item() <= 5e-5


def test_state_dict_keys_match_reference_checkpoint_format():
    from dino_tracker_b200.networks import DeltaDINO, TrackerHead
    d = DeltaDINO(channels=[3, 8, 12, 16, 24])
    keys = set(d.state_dict().keys())
    want = set(od.random_state_dict([3, 8, 12, 16, 24], torch.Generator().manual_seed(0)).keys())
    assert keys == want
    assert set(TrackerHead().state_dict().keys()) == {"cnn_refiner.0.weight", "cnn_refiner.0.bias",
                                                       "cnn_refiner.2.weight", "cnn_refiner.2.bias"}


@gpu
def test_tensor_core_convs_match_exact_path_and_oracle():
    """delta-DINO with the convolutions on wgmma (im2col + split-fp16 GEMM) vs the exact-fp32 CUDA-core path and
    the oracle, at a shape with ragged tiles (channels 16/24/40/72)."""
    from dino_tracker_b200 import Tracker
    channels = [3, 16, 24, 40, 72]
    H, W, T = 126, 154, 2
    geo = Geometry(H=H, W=W)
    sd = od.random_state_dict(channels, torch.Generator().manual_seed(33), last_std=0.05)
    video = synth.random_video(T, H, W, seed=34)
    dino = synth.random_features(T, channels[-1], geo.h, geo.w, seed=35)
    out = {}
    for prec in ("fp16x3", "fp32"):
        m = Tracker(video=video.to(DEV), dino_embed_video=dino, device=DEV, delta_channels=channels)
        m.delta_dino.conv_precision = prec
        m.delta_dino.load_state_dict(sd)
        m.cache_refined_embeddings()
        out[prec] = m.refined_features.cpu()
    ref = od.refined_features(video, dino, sd)
    e_tc = (out["fp16x3"] - ref).abs().max().item()
    e_ff = (out["fp32"] - ref).abs().max().item()
    print(f"delta-DINO max |diff| vs oracle: tensor {e_tc:.2e}, fp32 {e_ff:.2e}")
    assert e_ff <= 5e-5 and e_tc <= 5e-5
