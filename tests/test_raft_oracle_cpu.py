"""CPU suite: oracle/raft.py (the library's structure: per-frame encoders, a pair-batched update loop, the mask and the
upsampling after the last update only) equals torchvision's raft_large(a, b, n)[-1] in float64, and the library's weight
layout (dino_tracker_b200/raft.py conv_matrices) restates torchvision's convolutions."""
import pytest
import torch
import torch.nn.functional as F

tv = pytest.importorskip("torchvision.models.optical_flow")

from oracle import raft as oraft  # noqa: E402
from oracle.raft import seeded_model, textured_pair  # noqa: E402


@pytest.mark.parametrize("H,W", [(128, 128), (136, 248)])
def test_oracle_equals_torchvision_float64(H, W):
    m = seeded_model().double()
    a, b = textured_pair(H, W)
    a, b = a.double(), b.double()
    sd = {k: v for k, v in m.state_dict().items()}
    video = torch.cat([a, b])
    enc = oraft.encode(sd, video)
    with torch.no_grad():
        for n in (1, 3, 24):
            ref = oraft.torchvision_flow(m, a, b, n)
            # both directions in one batch of pairs
            ours = oraft.flows(sd, enc, [(0, 1), (1, 0)], n)
            ref_bwd = oraft.torchvision_flow(m, b, a, n)
            scale = max(ref.abs().max().item(), 1.0)
            assert (ours[0] - ref[0]).abs().max().item() <= 1e-9 * scale, n
            assert (ours[1] - ref_bwd[0]).abs().max().item() <= 1e-9 * scale, n
            if n == 24:
                assert ref.abs().max().item() >= 4.0   # the rescaled head moves points by several pixels


def test_lookup_channel_order_and_zero_padding():
    h, w = 16, 20
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    vol = (xs + 100 * ys)[None, None].expand(h * w, 1, h, w).contiguous()    # value = x + 100 y at every pixel's map
    levels = [vol] + [F.avg_pool2d(vol, 2, 2)]
    levels.append(F.avg_pool2d(levels[-1], 2, 2))
    levels.append(F.avg_pool2d(levels[-1], 2, 2))
    coords = torch.zeros(1, 2, h, w, dtype=torch.float64)
    coords[0, 0], coords[0, 1] = xs, ys
    coords[0, :, 0, 0] = torch.tensor([5.0, 7.0])           # pixel (0, 0) looks at (5, 7)
    coords[0, :, 0, 1] = torch.tensor([-30.0, 50.0])        # pixel (0, 1): every tap of every level outside the map
    feats = oraft.lookup(levels, coords)
    # torchvision's own CorrBlock agrees
    cb = tv.raft.CorrBlock(num_levels=4, radius=4)
    cb.corr_pyramid = levels
    assert torch.equal(cb.index_pyramid(coords), feats)
    # level 0, channel i * 9 + j samples (x + i - 4, y + j - 4): the first offset moves x
    for i in range(9):
        for j in range(9):
            assert feats[0, i * 9 + j, 0, 0].item() == pytest.approx((5 + i - 4) + 100 * (7 + j - 4))
    assert feats[0, :, 0, 1].abs().max().item() == 0.0


def test_conv_matrices_restate_torchvision_convolutions():
    from dino_tracker_b200 import raft
    m = seeded_model().double()
    mats = raft.conv_matrices(m.state_dict())
    assert len(mats) == 45
    x = torch.randn(1, 384, 9, 11, dtype=torch.float64)
    gru = m.update_block.recurrent_block.convgru1
    w, b = mats[37]                                          # [convz; convr] of the (1 x 5) GRU
    cols = F.unfold(x, (1, 5), padding=(0, 2))               # [1][ci * 5 + kx][pix] -> the library's (kx, ci) order
    cols = cols.view(1, 384, 5, -1).permute(0, 2, 1, 3).reshape(1, 5 * 384, -1)
    y = (w.double()[:256, :5 * 384] @ cols[0] + b.double()[:256, None]).view(256, 9, 11)
    ref = torch.cat([gru.convz(x), gru.convr(x)], dim=1)[0]
    assert (y - ref).abs().max().item() < 1e-5
    # the context encoder's stem with its BatchNorm folded
    stem = m.context_encoder.convnormrelu
    x = torch.rand(1, 3, 16, 16, dtype=torch.float64)
    w, b = mats[16]
    cols = F.unfold(x, 7, padding=3, stride=2).view(1, 3, 49, -1).permute(0, 2, 1, 3).reshape(147, -1)
    y = (w.double()[:64, :147] @ cols + b.double()[:64, None]).view(64, 8, 8)
    assert (y - stem[1](stem[0](x))[0]).abs().max().item() < 1e-5
