"""GPU: the foreground-mask kernels (row statistics, fused power pass, projection, nearest upsampling) and the fg / bg
trajectory split against the oracle on the same GPU and seed, against float64 PCA, at the shipped shapes and past 2^31
feature elements; and the whole preprocessing in one process."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import fg_masks as ofg
from oracle import make_golden_fg_masks as mgf
from oracle import trajectories as otr

from golden_util import GOLDEN_DIR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
THR = 0.6                 # preprocessing.yaml fg_mask_threshold


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(-1.0), b.nan_to_num(-1.0))


@pytest.mark.parametrize("T", [4, 50])
def test_pca_directions_and_masks_against_oracle(T):
    """476 x 854 frames (67 x 121 tokens), C = 1024, q = 3.  Directions: within 1 - |cos| <= 1e-5 of float64 PCA run from
    the same random start, with the signs of the oracle's fp32 torch.pca_lowrank on this GPU and seed.  Masks: identical
    to the oracle's except tokens whose float64 normalised component lies within 1e-4 of the threshold.  Measured on an
    H100: 1 - |cos| ~ 1e-14 at both T (the fp32 oracle's own run: ~2e-14), and no token of these planted features lies in
    the band or differs; the band stays at 1e-4 because it is the only allowance for last-bit ties at the threshold."""
    from dino_tracker_b200 import fg_masks as fgm
    h, w, C = 67, 121, 1024
    feats, plant = ofg.planted_features(T, h, w, C, seed=50 + T, noise=0.6, device=DEV)
    torch.manual_seed(7)
    mask, tm, V = fgm.fg_masks(feats, (476, 854), fg_mask_threshold=THR, return_all=True)
    torch.manual_seed(7)
    R = torch.randn(C, 3, device=DEV)
    torch.manual_seed(7)
    tm_o, V32, _ = ofg.fg_mask_tokens(feats, 3, True, THR)
    A64 = F.normalize(feats.double(), dim=-1).reshape(-1, C)
    V64 = ofg.pca_directions_from(A64, R.double())
    V64 = V64 * torch.sign((V64 * V32.double()).sum(0))            # the float64 run's own signs are not under test
    cos = (V.double() * V64).sum(0) / (V.double().norm(dim=0) * V64.norm(dim=0))
    sign32 = (V * V32).sum(0)
    print(f"T={T}: 1 - cos = {(1 - cos).tolist()}, fp32 oracle 1 - cos = "
          f"{(1 - (V32.double() * V64).sum(0) / (V32.double().norm(dim=0) * V64.norm(dim=0))).tolist()}")
    assert bool((1 - cos.abs() <= 1e-5).all()), cos
    assert bool((sign32 > 0).all()), sign32
    # masks: the float64 normalised first component decides which tokens are too close to call
    c64 = A64 @ V64[:, :1]
    t64 = ((c64 - c64.min()) / (c64.max() - c64.min())).reshape(T, h, w)
    near = (t64 - THR).abs() <= 1e-4
    diff = tm != tm_o
    print(f"T={T}: {int(near.sum())} tokens within 1e-4 of the threshold, {int(diff.sum())} differ, "
          f"{int((diff & ~near).sum())} of them outside the band; fg fraction {float(tm.float().mean()):.3f}")
    assert not bool((diff & ~near).any())
    assert torch.equal(mask, fgm.upsample_mask(tm, (476, 854)))
    # the reference's signature and return type
    torch.manual_seed(7)
    got = fgm.get_fg_mask_from_pca(feats, (476, 854), fg_mask_threshold=THR)
    assert got.dtype == np.float32 and got.shape == (T, 476, 854)
    assert np.array_equal(got, (mask > 0).float().cpu().numpy())


def test_fg_mask_fixture_on_gpu():
    """The reference's CPU mask of the small planted case, reproduced by the kernels from the reference's CPU start.  The
    sign of a singular vector is the SVD backend's convention (LAPACK on the CPU, cuSOLVER here) and decides which side
    of the first component falls below the threshold, so the kernels' mask is the reference's or its exact complement;
    same-device sign parity is checked against the oracle above."""
    from dino_tracker_b200 import fg_masks as fgm
    cfg = mgf.FG_CASE
    feats, _ = mgf.fg_case_inputs()
    torch.manual_seed(cfg["torch_seed"])
    R = torch.randn(cfg["C"], cfg["q"])                            # pca_lowrank's draw on the CPU
    mask = fgm.fg_masks(feats.to(DEV), (cfg["H"], cfg["W"]), q=cfg["q"], fg_mask_threshold=cfg["threshold"], R=R.to(DEV))
    ref = np.load(os.path.join(GOLDEN_DIR, "fg_mask_small.npz"))["mask"]
    got = (mask > 0).cpu().numpy().astype(np.uint8)
    assert np.array_equal(got, ref) or np.array_equal(got, 1 - ref)


@pytest.mark.parametrize("hw", [(67, 121, 476, 854), (13, 17, 98, 126), (9, 12, 61, 86), (7, 5, 23, 19)])
def test_upsample_matches_interpolate_nearest(hw):
    from dino_tracker_b200 import fg_masks as fgm
    h, w, H, W = hw
    tm = torch.rand(3, h, w, generator=torch.Generator().manual_seed(h * w)) < 0.5
    ref = F.interpolate(tm.to(DEV)[None].float(), size=(H, W), mode="nearest")[0]
    ref_cpu = F.interpolate(tm[None].float(), size=(H, W), mode="nearest")[0]
    got = fgm.upsample_mask(tm.to(DEV), (H, W))
    assert torch.equal(got.cpu(), (ref.cpu() * 255).to(torch.uint8))
    assert torch.equal(ref.cpu(), ref_cpu)


def test_large_shape_past_2_31_elements():
    """T = 300 frames of 67 x 121 tokens at C = 1024: 2.49e9 elements, past 2^31.  The plant is far from the threshold, so
    the mask is the planted disc exactly (on the side of the first component that the SVD's sign puts below the
    threshold: the disc or its complement).  Two runs give the same bits, and so do two power passes."""
    from dino_tracker_b200 import fg_masks as fgm
    T, h, w, C = 300, 67, 121, 1024
    feats, plant = ofg.planted_features(T, h, w, C, seed=300, noise=0.3, device=DEV)
    assert feats.numel() > 2 ** 31
    runs = []
    for _ in range(2):
        torch.manual_seed(11)
        mask, tm, V = fgm.fg_masks(feats, (476, 854), fg_mask_threshold=THR, return_all=True)
        runs.append((mask, tm, V))
    tm = runs[0][1]
    side = "disc" if torch.equal(tm, plant) else "complement"
    print(f"T=300: mask = planted {side}, fg fraction {float(tm.float().mean()):.3f}")
    assert torch.equal(tm, plant) or torch.equal(tm, ~plant)
    assert all(torch.equal(a, b) for a, b in zip(runs[0], runs[1]))
    passes = fgm.PcaPasses(feats.view(-1, C))
    P = torch.randn(C, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    X1, W1 = passes.power(P)
    X2, W2 = passes.power(P)
    assert torch.equal(X1, X2) and torch.equal(W1, W2)
    # the last rows (offsets past 2^31) are projected like the first
    rows = feats.view(-1, C)[-5:].double()
    x = (rows * passes.s[-5:, None].double() - passes.c.double()) @ P.double()
    assert (X1[-5:].double() - x).abs().max().item() <= 1e-5 * x.abs().max().item()


def test_argument_errors():
    from dino_tracker_b200 import _lib
    from dino_tracker_b200 import fg_masks as fgm
    with pytest.raises(_lib.DinotrkError):
        fgm.PcaPasses(torch.ones(64, 6, device=DEV))                   # C % 4 != 0
    with pytest.raises(_lib.DinotrkError):
        fgm.PcaPasses(torch.ones(64, 1540, device=DEV))                # C > 1536
    with pytest.raises(ValueError):
        fgm.fg_masks(torch.ones(1, 4, 4, 8, device=DEV), (8, 8), q=5)
    with pytest.raises(ValueError):
        fgm.get_fg_mask_from_pca(torch.ones(1, 4, 4, 8, device=DEV), (8, 8), interpolation="bilinear")


def test_split_smooth_flows_full_size():
    """Trajectories chained from seeded smooth flows at 476 x 854, T = 50, split by 50 disc masks: fg and bg equal the
    oracle's bit for bit."""
    from dino_tracker_b200.fg_masks import split_trajectories
    from dino_tracker_b200.trajectories import chain_trajectories
    T, H, W = 50, 476, 854
    fwd, bwd, _ = otr.stack_flows(otr.smooth_flows(T, H, W, seed=91, amplitude=3.0, device=DEV, noise=False), T)
    traj = chain_trajectories(fwd, bwd, None, 1.0, 2)
    _, masks = ofg.split_case_inputs(1, T, H, W, seed=92)
    masks = masks.to(DEV)
    fg, bg = split_trajectories(traj, masks)
    print(f"split: {traj.shape[0]} trajectories, {fg.shape[0]} fg")
    assert fg.shape[0] > 1000 and bg.shape[0] > 1000
    assert _same(fg, ofg.mask_filter(traj, masks))
    assert _same(bg, ofg.mask_filter(traj, masks, filter_bg=True))


def test_split_fixture_ties_last_frame_and_errors():
    """The reference's split of the fixture (exact .5 start positions), starts at frame T - 1, and trajectories that
    start outside the frame or never start: DinotrkError, no fault, and the library keeps working."""
    from dino_tracker_b200 import _lib
    from dino_tracker_b200.fg_masks import split_trajectories
    cfg = mgf.SPLIT_CASE
    traj, masks = ofg.split_case_inputs(cfg["N"], cfg["T"], cfg["H"], cfg["W"], cfg["seed"])
    ref = np.load(os.path.join(GOLDEN_DIR, "traj_split_small.npz"))
    fg, bg = split_trajectories(traj.to(DEV), masks.to(DEV))
    assert np.array_equal(fg.cpu().numpy(), ref["fg"], equal_nan=True)
    assert np.array_equal(bg.cpu().numpy(), ref["bg"], equal_nan=True)
    last = torch.full((4, cfg["T"], 2), float("nan"))
    last[:, -1] = torch.tensor([[10.5, 3.5], [11.5, 4.5], [853.0, 475.0], [0.0, 0.0]])
    m = masks.clone()
    m[-1] = 0
    m[-1, 4, 12] = 7                                               # (11.5, 4.5) rounds to (12, 4)
    fg, bg = split_trajectories(last.to(DEV), m.to(DEV))
    assert _same(fg.cpu(), ofg.mask_filter(last, m)) and fg.shape[0] == 1
    assert _same(bg.cpu(), ofg.mask_filter(last, m, filter_bg=True))
    for bad in ([[853.6, 10.0]], [[-0.6, 10.0]], [[10.0, 475.5]], [[float("nan"), float("nan")]]):
        t = last.clone()
        t[2, -1] = torch.tensor(bad[0])
        with pytest.raises(_lib.DinotrkError):
            split_trajectories(t.to(DEV), m.to(DEV))
    torch.cuda.synchronize()
    fg2, _ = split_trajectories(last.to(DEV), m.to(DEV))
    assert torch.equal(fg2.nan_to_num(-1), fg.nan_to_num(-1))


def test_preprocess_video_writes_the_reference_files(tmp_path):
    """preprocess_video on a small video with random ViT weights and a seeded flow_fn: the reference's files, the masks
    as JPEG frames, fg = the split of the masks read back from them, fg + bg = all trajectories."""
    from oracle import vit as ovit
    from dino_tracker_b200 import DinoV2Features
    from dino_tracker_b200.fg_masks import load_masks
    from dino_tracker_b200.pipeline import preprocess_video
    H, W, T, D = 98, 126, 3, 64
    g = torch.Generator().manual_seed(8)
    vit = DinoV2Features(ovit.random_state_dict(2, D, g, n_pos=4, std=0.08), heads=1, layer=1, device=DEV)
    mask_vit = DinoV2Features(ovit.random_state_dict(2, D, g, n_pos=4, std=0.08), heads=1, layer=1, device=DEV)
    flow = otr.smooth_flows(T, H, W, seed=83, amplitude=6.0, integer=True, device=DEV)
    video = torch.arange(T, dtype=torch.float32).view(T, 1, 1, 1).expand(T, 3, H, W).contiguous() / 8
    video = video + 0.05 * torch.rand(T, 3, H, W, generator=torch.Generator().manual_seed(9))

    def flow_fn(a, b):   # the frames carry their index in their mean value
        ia, ib = (x.mean(dim=(1, 2, 3)).sub(0.025).mul(8).round().long().tolist() for x in (a, b))
        return torch.stack([flow(i, j) for i, j in zip(ia, ib)])

    torch.manual_seed(3)
    traj, fg, bg, masks = preprocess_video(video, vit, mask_vit, str(tmp_path), flow_fn=flow_fn, device=DEV)
    for f in ("of_trajectories/trajectories.pt", "of_trajectories/fg_trajectories.pt", "of_trajectories/bg_trajectories.pt",
              "of_trajectories/trajectories_wo_direct_filter.pt", "dino_embeddings/dino_embed_video.pt",
              "dino_best_buddies/dino_best_buddies.pt", "dino_best_buddies/dino_best_buddies_filtered.pt",
              *[f"masks/{k:05d}.jpg" for k in range(T)]):
        assert os.path.exists(tmp_path / f), f
    saved = torch.load(tmp_path / "of_trajectories/trajectories.pt")
    assert _same(saved, traj.cpu()) and saved.shape[0] > 0
    reread = torch.from_numpy(load_masks(tmp_path / "masks", H, W))
    assert torch.equal(reread, masks.cpu())
    fg_file = torch.load(tmp_path / "of_trajectories/fg_trajectories.pt")
    bg_file = torch.load(tmp_path / "of_trajectories/bg_trajectories.pt")
    assert _same(fg_file, ofg.mask_filter(saved, reread)) and _same(bg_file, ofg.mask_filter(saved, reread, filter_bg=True))
    assert fg_file.shape[0] + bg_file.shape[0] == saved.shape[0]
    # a second run finds the masks and keeps them
    mtime = os.path.getmtime(tmp_path / "masks/00000.jpg")
    preprocess_video(video, vit, mask_vit, str(tmp_path), flow_fn=flow_fn, device=DEV)
    assert os.path.getmtime(tmp_path / "masks/00000.jpg") == mtime
