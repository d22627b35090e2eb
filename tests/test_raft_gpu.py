"""GPU suite: the library's RAFT-large (dino_tracker_b200/raft.py) against torchvision's raft_large run in float64 on
the same GPU, with seeded weights whose flow head is rescaled so that 24 updates move points by several pixels.

Bars, pinned from the H100 run (numbers in DESIGN.md 4.8): the library's max |flow error| is at most 10x that of
torchvision in fp32 with TF32 off (measured 2x to 7x) and at most a tenth of torchvision's default with cuDNN TF32 on
(measured over 100x below it); both are printed."""
import warnings

import pytest
import torch

from oracle import raft as oraft

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FP32_BAR = 10    # library error at most this multiple of the fp32 error (floor 1e-4 px)


@pytest.fixture(scope="module")
def model():
    return oraft.seeded_model().to(DEV)


@pytest.fixture(scope="module")
def lib_raft(model):
    from dino_tracker_b200.raft import RaftLarge
    return RaftLarge(model, device=DEV)


def padded(x):
    """raft_flow_fn's replicate padding to a multiple of 8 ("sintel": the extra row / column split evenly)."""
    ht, wd = x.shape[-2:]
    ph, pw = (((ht // 8) + 1) * 8 - ht) % 8, (((wd // 8) + 1) * 8 - wd) % 8
    pad = [pw // 2, pw - pw // 2, ph // 2, ph - ph // 2]
    return torch.nn.functional.pad(x, pad, mode="replicate"), pad


def tv_flows(model, a, b, ns, dtype, tf32=False):
    """torchvision raft_large on padded frames in ``dtype``, cropped back: the flows after each number of updates in
    ``ns``, from one run of max(ns) updates."""
    (ap, pad), (bp, _) = padded(a), padded(b)
    m = model if dtype == torch.float32 else _copy(model, dtype)
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
    try:
        fs = oraft.torchvision_flows(m, ap.to(dtype), bp.to(dtype), max(ns))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    return [fs[n - 1][..., pad[2]:fs[n - 1].shape[-2] - pad[3], pad[0]:fs[n - 1].shape[-1] - pad[1]].double() for n in ns]


def tv_flow(model, a, b, n, dtype, tf32=False):
    """torchvision raft_large on padded frames in ``dtype``, cropped back."""
    return tv_flows(model, a, b, (n,), dtype, tf32)[0]


_copies = {}


def _copy(model, dtype):
    key = (id(model), dtype)
    if key not in _copies:
        import copy
        _copies[key] = copy.deepcopy(model).to(dtype)
    return _copies[key]


def pair(H, W, shift=(2.5, -1.5)):
    a, b = oraft.textured_pair(H, W, shift)
    return a.to(DEV), b.to(DEV)


@pytest.mark.parametrize("H,W", [(128, 128), (136, 248), (476, 854)])
def test_flows_against_torchvision_float64(model, lib_raft, H, W):
    a, b = pair(H, W)
    enc = lib_raft.encode(torch.cat([a, b]))
    assert enc.hi is not None, "fmaps outside the split's range: this test is meant for the F16X3 path"
    bad = []
    for n in (1, 12, 24):
        ours = lib_raft.flows(enc, [(0, 1), (1, 0)], n).double()
        for d, (x, y) in enumerate(((a, b), (b, a))):
            ref = tv_flow(model, x, y, n, torch.float64)
            e_lib = (ours[d] - ref[0]).abs().max().item()
            e_f32 = (tv_flow(model, x, y, n, torch.float32) - ref).abs().max().item()
            e_tf32 = (tv_flow(model, x, y, n, torch.float32, tf32=True) - ref).abs().max().item()
            print(f"RAFT {H}x{W} n={n} dir={d}: max|flow|={ref.abs().max().item():.3f}  library {e_lib:.3e}  "
                  f"torchvision fp32 {e_f32:.3e}  fp32+TF32 {e_tf32:.3e}")
            if e_lib > max(FP32_BAR * e_f32, 1e-4) or e_lib > 0.1 * e_tf32:
                bad.append((n, d, e_lib, e_f32))
            if n == 24:
                assert ref.abs().max().item() >= 4.0
                # some points end outside the frame: their lookups sample outside the correlation maps
                ys, xs = torch.meshgrid(torch.arange(H, device=DEV), torch.arange(W, device=DEV), indexing="ij")
                tx, ty = xs + ref[0, 0], ys + ref[0, 1]
                assert bool(((tx < 0) | (tx > W - 1) | (ty < 0) | (ty > H - 1)).any())
    assert not bad, bad


def test_same_bits_across_runs_and_batches(lib_raft):
    T, H, W = 5, 136, 248
    frames = torch.cat([pair(H, W, (0.7 * t, -0.4 * t))[1] for t in range(T)])
    enc = lib_raft.encode(frames)
    pairs = [(i, j) for i in range(T) for j in range(T) if i != j][:16]
    f16 = lib_raft.flows(enc, pairs, 12)
    assert torch.equal(f16, lib_raft.flows(enc, pairs, 12))                   # two runs
    enc2 = lib_raft.encode(frames)
    assert torch.equal(enc.fmap, enc2.fmap) and torch.equal(enc.ctx, enc2.ctx)
    for k in (0, 7, 15):                                                      # batches of 1, 2 and 16
        assert torch.equal(lib_raft.flows(enc, [pairs[k]], 12)[0], f16[k])
        assert torch.equal(lib_raft.flows(enc, [pairs[k], pairs[(k + 5) % 16]], 12)[0], f16[k])
    # a memory budget of one pair splits the call; the bits do not change
    from dino_tracker_b200.raft import RaftLarge
    small = RaftLarge.__new__(RaftLarge)
    small.__dict__.update(lib_raft.__dict__)
    small.memory_budget = 1
    assert small.batch_pairs(H, W) == 1
    assert torch.equal(small.flows(enc, pairs, 12), f16)
    # flow_fn contract: a batch of frame pairs
    assert torch.equal(lib_raft(frames[:2], frames[2:4]), lib_raft.flows(enc, [(0, 2), (1, 3)], 24))


def oracle_flows(model, enc, pairs, n, dtype=torch.float64):
    """oracle/raft.py in ``dtype`` (TF32 off) on the library's own encodings (the update loop only)."""
    sd = {k: v.to(dtype) for k, v in model.state_dict().items()}
    h, w = -(-enc.H // 8), -(-enc.W // 8)
    chw = lambda x: x.to(dtype).view(x.shape[0], h, w, -1).permute(0, 3, 1, 2)
    ctx = chw(enc.ctx)
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return oraft.flows(sd, (chw(enc.fmap), ctx[:, :128], ctx[:, 128:]), pairs, n).double()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


@pytest.mark.parametrize("case", ["tiny_tokens", "large"])
def test_correlation_paths_against_float64_on_the_same_encoding(model, lib_raft, case):
    """The update loop on given encodings, against oracle/raft.py in float64 on the same encodings (bar: FP32_BAR times
    the oracle's own fp32 error), so the result depends on the correlations:
      tiny_tokens: a few tokens scaled by 2^-20 put the fmaps outside the split's faithful range while the other
        correlations stay O(1): the exact-fp32 level 0 and the F16X3 level 0 both give the float64 flows;
      large: fmaps scaled by 2^5, correlations up to ~1e5 (beyond fp16): the per-row scaled lookup operand keeps them
        finite and accurate."""
    from dino_tracker_b200 import _lib
    from dino_tracker_b200.raft import RaftEncoding
    H, W = 136, 248
    a, b = pair(H, W)
    enc = lib_raft.encode(torch.cat([a, b]))
    fmap = enc.fmap.clone()
    if case == "tiny_tokens":
        fmap[1, :3] *= 2.0 ** -20
    else:
        fmap *= 2.0 ** 5
    norms = fmap.norm(dim=-1).contiguous()
    with torch.cuda.device(DEV):
        st = _lib.stream_ptr()
        ok = _lib.split_range(fmap, norms, st)[2]
        hi, lo = _lib.split_fp16(fmap, st)
    assert ok == (case == "large")
    pairs = [(0, 1), (1, 0)]
    plain = RaftEncoding(fmap, enc.ctx, None, None, H, W)
    ref = oracle_flows(model, plain, pairs, 12)
    e_f32 = (oracle_flows(model, plain, pairs, 12, torch.float32) - ref).abs().max().item()
    paths = {"F16X3": RaftEncoding(fmap, enc.ctx, hi, lo, H, W)}
    if case == "tiny_tokens":
        paths["exact-fp32"] = RaftEncoding(fmap, enc.ctx, None, None, H, W)
    for name, e in paths.items():
        f = lib_raft.flows(e, pairs, 12).double()
        assert bool(torch.isfinite(f).all())
        err = (f - ref).abs().max().item()
        print(f"RAFT {case} {name}: max|flow|={ref.abs().max().item():.2f}  library vs float64 {err:.3e}  "
              f"oracle fp32 {e_f32:.3e}")
        assert err <= max(FP32_BAR * e_f32, 1e-4)


def test_out_of_range_encoding_warns(model):
    """fmaps scaled by 2^-12 fall outside the split's faithful range: encode warns and leaves no split (the flows then
    run on the exact-fp32 level 0, checked above)."""
    import copy

    from dino_tracker_b200.raft import RaftLarge
    m = copy.deepcopy(model)
    with torch.no_grad():
        m.feature_encoder.conv.weight.mul_(2.0 ** -12)
        m.feature_encoder.conv.bias.mul_(2.0 ** -12)
    lr = RaftLarge(m, device=DEV)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        enc = lr.encode(torch.cat(pair(136, 248)))
    assert enc.hi is None and any("faithful range" in str(x.message) for x in w)
    assert bool(torch.isfinite(lr.flows(enc, [(0, 1)], 3)).all())


def test_argument_errors_raise_before_any_launch(lib_raft):
    from dino_tracker_b200 import _lib
    enc = lib_raft.encode(torch.cat(pair(128, 128)))
    with pytest.raises(_lib.DinotrkError):
        lib_raft.flows(enc, [(0, 2)])                 # frame index out of range
    with pytest.raises(_lib.DinotrkError):
        lib_raft.encode(torch.rand(1, 3, 96, 128, device=DEV))   # 1/8 grid below 16 x 16


def _round_trip(f, b):
    """|f(p) + b(p + f(p))| per pixel (bilinear, border): the consistency the chaining thresholds."""
    H, W = f.shape[-2:]
    ys, xs = torch.meshgrid(torch.arange(H, device=f.device, dtype=f.dtype), torch.arange(W, device=f.device, dtype=f.dtype),
                            indexing="ij")
    grid = torch.stack([(xs + f[0]) / (W - 1) * 2 - 1, (ys + f[1]) / (H - 1) * 2 - 1], -1)[None]
    bs = torch.nn.functional.grid_sample(b[None], grid, align_corners=True, padding_mode="border")[0]
    return (f + bs).norm(dim=0)


def _start_keys(traj):
    """{(start frame, x, y)} of trajectories [M][T][2]."""
    valid = ~torch.isnan(traj[..., 0])
    s = valid.float().argmax(dim=1)
    xy = traj[torch.arange(traj.shape[0], device=traj.device), s].round().long()
    return set(zip(s.tolist(), xy[:, 0].tolist(), xy[:, 1].tolist()))


def test_extract_trajectories_with_library_raft(model, lib_raft):
    """The chaining of extract_trajectories (direct filter on) on a textured video with known sub-pixel motion, with the
    library's flows and with torchvision fp32 flows of the same weights.  The surviving start pixels may differ only
    through threshold decisions (round trip against 1.5 px consecutive, 2.5 px direct) that lie within the two flows'
    measured difference of the threshold: each such decision can end at most one trajectory and start one."""
    from dino_tracker_b200.trajectories import chain_trajectories, video_flows
    lib = lib_raft
    T, H, W = 10, 128, 160
    video = torch.cat([oraft.textured_pair(H, W, (0.6 * t, 0.35 * t))[1] for t in range(T)]).to(DEV)

    def tv_fn(a, b):
        return tv_flow(model, a, b, 24, torch.float32).float()

    lf, lb, ldir = video_flows(video, lib, True, DEV)
    tf, tb, tdir = video_flows(video, tv_fn, True, DEV)
    dl = {s: ldir(s) for s in range(T - 1)}
    dt = {s: tdir(s) for s in range(T - 1)}
    near = 0
    e = max((lf - tf).abs().max().item(), (lb - tb).abs().max().item())
    for i in range(T - 1):    # consecutive round trips, both directions
        for f, b in ((tf[i], tb[i]), (tb[i], tf[i])):
            near += int(((_round_trip(f, b) - 1.5).abs() <= 2 * e).sum())
    for s in range(T - 1):
        ed = max((dl[s][0] - dt[s][0]).abs().max().item(), (dl[s][1] - dt[s][1]).abs().max().item())
        e = max(e, ed)
        for k in range(T - 1 - s):
            near += int(((_round_trip(dt[s][0][k], dt[s][1][k]) - 2.5).abs() <= 2 * ed).sum())
    kw = dict(threshold=1.5, min_trajectory_length=2, direct_flow_threshold=2.5)
    ours = _start_keys(chain_trajectories(lf, lb, lambda s: dl[s], **kw))
    ref = _start_keys(chain_trajectories(tf, tb, lambda s: dt[s], **kw))
    diff = len(ours ^ ref)
    print(f"RAFT trajectories: library {len(ours)}, torchvision fp32 {len(ref)}, differing starts {diff}, "
          f"decisions within 2 x {e:.2e} px of a threshold {near}")
    assert len(ref) > 20     # random-weight flows are rarely round-trip consistent: 57 survive at this seed
    assert diff <= 2 * near
