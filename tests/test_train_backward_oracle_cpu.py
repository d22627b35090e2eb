"""The float64 reference of the tracker node's reverse pass (tests/track_reverse.py), pinned on the CPU.

Autograd through the oracle chain in float64 -- with the arg-max, the stability branch and the ReLU of the maps pinned
to the fp32 oracle's own decisions -- must agree with autograd through the same chain in fp32 element by element,
within kappa u M (M from ``abs_reverse``).  This is what tests/test_train_backward_gpu.py relies on: the float64
oracle computes the same function as the fp32 one (the trilinear weights stay fp32, leak included), and M dominates
the gradient it bounds.
"""
import pytest
import torch

from oracle import synth
from oracle.tracker import Geometry

import track_reverse as tr

# fp32 autograd on the CPU against float64, in units of u M: 0.16 ("well") and 9.6 ("default": logits ~1e3) measured;
# pinned with over 3x headroom
KAPPA_FP32_ORACLE = 32.0


@pytest.mark.parametrize("kind", ["well", "default"])
def test_float64_oracle_reverse_agrees_with_fp32(kind):
    geo = Geometry(H=98, W=126)
    N, C, B = 4, 32, 48
    feats, _ = synth.shifted_field_features(N, C, geo.h, geo.w, seed=91, noise=0.2, max_shift=2)
    wts = tr.normalized_weights(synth.head_weights(kind, seed=91))
    gen = torch.Generator().manual_seed(92)
    pts_px = torch.rand(B, 2, generator=gen) * torch.tensor([geo.W - 1.0, geo.H - 1.0])
    src, tgt = torch.randint(0, N, (B,), generator=gen), torch.randint(0, N, (B,), generator=gen)
    gout = tr.draw_grad_out(B, gen)
    fs = torch.arange(N, dtype=torch.int32)
    pts_n = tr.sampling_points(torch.cat([pts_px, src[:, None].float()], 1), geo)
    with torch.no_grad():
        _, aux0 = tr.oracle_coords(feats, pts_n, tgt, fs, wts, geo)
        relu_mask = tr.ot.corr_maps(tr.ot.sample_descriptors(feats, pts_n, fs), feats, tgt, frames_set=fs) > 0
    amax, fb = aux0["argmax"], aux0["fallback"]
    assert fb.any() == (kind == "default"), "the 'default' head puts maps on the stability branch, 'well' none"
    g32f, g32w, out32, _ = tr.reference_gradients(feats, pts_n, tgt, fs, wts, geo, gout, amax, fb, relu_mask)
    g64f, g64w, out64, aux = tr.reference_gradients(feats.double(), pts_n, tgt, fs, wts, geo, gout, amax, fb, relu_mask)
    moved = int(((aux["own_argmax"] != amax) | (aux["own_fallback"] != fb)).sum())
    M, Mw, _ = tr.abs_reverse(feats, pts_n, tgt, fs, wts, geo, gout, amax, fb, relu_mask, KAPPA_FP32_ORACLE,
                             full_softmax=True)
    assert (g64f.abs() <= M).all() and (g64w.abs() <= Mw).all(), "M must dominate the gradient it bounds"
    for name, got, ref, m in (("d/dfeats", g32f, g64f, M), ("d/dw", g32w, g64w, Mw)):
        err = (got.double() - ref).abs()
        ratio = tr.worst_ratio(err, tr.U * m)
        print(f"[{kind} {name}] worst error / (u M) = {ratio:.4f}; float64 decisions differing from fp32: {moved}")
        assert ratio <= KAPPA_FP32_ORACLE, (name, ratio)
