"""GPU suite: the library's training-batch sampler (dino_tracker_b200/sampler.py, dinotrk_sampler_*) against the oracle's
restatement of the reference (oracle/sampler.py) on the same GPU under the same seed: identical sample dicts (values,
dtypes, shapes, devices), in both modes, across 64-bit element offsets, and through one whole training iteration."""
import pytest
import torch

from oracle import make_golden_sampler as mg
from oracle import sampler as osm

pytestmark = pytest.mark.gpu

DEV = "cuda"
KEYS = mg.KEYS


def normalizer(T):
    return osm.RangeNormalizer(shapes=(mg.W, mg.H, T), device=DEV)


def run(cls, fg, bg, T, calls, seed, batch=512, num_frames=4, ratio=0.5, ops=None, **kw):
    torch.manual_seed(seed)
    s = cls(batch_size=batch, range_normalizer=normalizer(T), dst_range=(-1, 1), fg_trajectories=fg, bg_trajectories=bg,
            fg_traj_ratio=ratio, num_frames=num_frames, **kw)
    out = []
    for op in ops or ["call"] * calls:
        if op == "next":
            s.load_next_batch()
        else:
            out.append(s())
    return out


def assert_same(lib, ref):
    assert len(lib) == len(ref)
    for i, (a, b) in enumerate(zip(lib, ref)):
        assert set(a) == set(b) == set(KEYS)
        for k in KEYS:
            x, y = a[k], b[k]
            assert x.dtype == y.dtype and x.shape == y.shape and x.device == y.device, (i, k, x.dtype, y.dtype, x.shape, y.shape)
            assert torch.equal(x, y), (i, k)


def both(fg, bg, T, calls, seed, **kw):
    from dino_tracker_b200 import sampler as sm
    lib = run(sm.DinoTrackerSampler, fg, bg, T, calls, seed, **kw)
    ref = run(osm.DinoTrackerSampler, fg, bg, T, calls, seed, **kw)
    assert_same(lib, ref)
    return lib


def test_train_shape_200_calls():
    """train.yaml's batch (512, 4 frames, fg ratio 0.5) on about 1M trajectories at T = 50."""
    fg = mg.make_trajectories(600_000, 50, 31).to(DEV)
    bg = mg.make_trajectories(400_000, 50, 32).to(DEV)
    out = both(fg, bg, 50, 200, seed=33)
    assert all(o["t1_points"].shape == (512, 3) for o in out)


@pytest.mark.parametrize("T", [3, 32, 33, 64, 65])
def test_small_shapes(T):
    """T = 3 has fewer frames than num_frames; 32 / 33 / 64 / 65 straddle the word boundaries of the frame bits."""
    fg = mg.make_trajectories(700, T, 40 + T).to(DEV)
    bg = mg.make_trajectories(900, T, 80 + T).to(DEV)
    both(fg, bg, T, 30, seed=T, batch=128)


def test_fg_set_of_three():
    T = 12
    fg = torch.rand(3, T, 2) * 100                 # three rows valid at every frame: always 3 candidates
    bg = mg.make_trajectories(2000, T, 6)
    out = both(fg.to(DEV), bg.to(DEV), T, 30, seed=7, batch=64)
    assert all(o["t1_points"].shape[0] == 3 + 32 for o in out)


def test_windowed_mode():
    """keep_in_cpu: the fixture's windowed case (three load_next_batch calls: fg windows 0, 1, 2, 0) from CPU and from
    CUDA inputs; the device holds less than the reference's two windows."""
    from dino_tracker_b200 import sampler as sm
    c = mg.CASES["windowed"]
    fg, bg = mg.case_inputs("windowed")
    kw = dict(batch=c["batch"], num_frames=c["num_frames"], ratio=c["ratio"], ops=c["ops"], keep_in_cpu=True)
    ref = run(osm.DinoTrackerSampler, fg, bg, c["T"], 0, c["seed"], window_device=DEV, **kw)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    lib_sampler = []
    lib = run(lambda **a: lib_sampler.append(sm.DinoTrackerSampler(**a)) or lib_sampler[-1], fg, bg, c["T"], 0, c["seed"],
              **kw)
    held = torch.cuda.memory_allocated() - base
    assert_same(lib, ref)
    assert held < 2 * osm.MAX_TRAJ_SIZE * c["T"] * (8 + 1), held
    assert lib_sampler[0].fg.rows.device.type == "cpu" and lib_sampler[0].fg.rows.is_pinned()
    lib2 = run(sm.DinoTrackerSampler, fg.to(DEV), bg.to(DEV), c["T"], 0, c["seed"], **kw)
    assert_same(lib2, ref)


def test_64bit_offsets():
    """A set of N * T * 2 > 2^31 elements whose valid rows lie mostly past element 2^31."""
    T, N = 64, 17_200_000
    assert N * T * 2 > 2 ** 31
    big = torch.full((N, T, 2), float("nan"), device=DEV)
    tail = 16_900_000
    big[tail:] = torch.rand(N - tail, T, 2, device=DEV) * 800
    big[:tail:1000] = torch.rand(len(range(0, tail, 1000)), T, 2, device=DEV) * 800
    big[-5:, ::2, 1] = float("nan")
    bg = mg.make_trajectories(5000, T, 9).to(DEV)
    out = both(big, bg, T, 5, seed=11)
    assert all(o["t1_points"].shape == (512, 3) for o in out)


def test_argument_errors_raise_before_any_launch():
    from dino_tracker_b200 import _lib
    from dino_tracker_b200 import sampler as sm
    ok = mg.make_trajectories(100, 8, 1).to(DEV)
    rn = normalizer(8)

    def make(fg, **kw):
        return sm.DinoTrackerSampler(8, rn, (-1, 1), fg_trajectories=fg, bg_trajectories=ok, num_frames=4, **kw)

    for bad, exc in ((ok.double(), TypeError), (ok[..., :1].contiguous(), ValueError), (ok[0], ValueError),
                     (ok.cpu(), _lib.DinotrkError), (ok[:1], ValueError), ([[0.0]], TypeError)):
        before = _lib.launch_count()
        with pytest.raises(exc):
            make(bad)
        assert _lib.launch_count() == before, exc
    one_valid = torch.full((50, 8, 2), float("nan"), device=DEV)
    one_valid[7] = 1.0
    one_valid[8, 3] = 2.0                                      # a single-step row
    before = _lib.launch_count()
    with pytest.raises(ValueError, match="1 valid"):
        make(one_valid)
    assert _lib.launch_count() - before == 2                    # the count and its scan; nothing is emitted


# the backward's float atomics (embedding gradients of the sampled descriptors) add in a run-dependent order; parameter
# gradients of the same iteration run twice differ by up to 7.5e-5 of each tensor's largest entry (measured on an H100;
# library against oracle sampler: 6.9e-5)
ITER_GRAD_SPREAD = 3e-4


def test_whole_iteration_library_sampler_against_oracle_sampler():
    """dino_tracker.py:405-427 at train.yaml's shape (50 frames of 476 x 854, C = 1024, shipped delta-DINO widths, batch
    512 of 4 frames, both contrastive terms): the library sampler and the oracle sampler feed the drop-in Tracker and the
    library's contrastive losses under the same seed; samples and loss bits are identical.  The parameter gradients agree
    to the run-to-run spread of the backward's float atomics (the same route run twice shows it)."""
    from test_delta_train_gpu import SHIPPED, _sd
    from dino_tracker_b200 import Tracker
    from dino_tracker_b200 import contrastive as c
    from dino_tracker_b200 import sampler as sm
    from oracle import contrastive as oc
    from oracle import make_golden_contrastive as mgc
    from oracle import synth
    H, W, T, C = 476, 854, 50, 1024
    h, w = (H - 14) // 7 + 1, (W - 14) // 7 + 1
    feats = synth.random_features(T, C, h, w, seed=300)
    video = synth.random_video(T, H, W, seed=301).to(DEV)
    m = Tracker(video=video, dino_embed_video=feats, device=DEV, delta_channels=SHIPPED)
    m.tracker_head.load_state_dict(synth.head_weights("well", seed=302))
    m.delta_dino.load_state_dict(_sd(SHIPPED, 303, last_std=0.02))
    m.train()
    cfg = dict(mgc.CONFIG, cl_points_per_pair=256, lambda_cl_dino_bb=0.00025, lambda_cl_ref_bb=0.00005,
               lambda_emb_norm=0.0001, lambda_angle=0.0001)
    g = torch.Generator().manual_seed(304)
    masks = torch.zeros(T, H, W)
    masks[:, 120:360, 250:600] = 1
    coords = oc.get_vit_feature_coords_from_mask(H, W, 7, 14)
    bb = {}
    for s in range(T):
        for t in range(T):
            if s != t:
                n = 300
                bb[f"{s}_{t}"] = {"source_coords": coords[torch.randperm(h * w, generator=g)[:n]],
                                  "target_coords": coords[torch.randint(h * w, (n,), generator=g)],
                                  "cos_sims": torch.rand(n, generator=g) * 0.6 + 0.4, "r": torch.rand(n, generator=g) * 0.4}
    tr = type("Trainer", (), {})()
    tr.config, tr.fg_masks, tr.dino_bb_pairs = cfg, masks, bb
    fg = mg.make_trajectories(300_000, T, 305).to(DEV)
    bg = mg.make_trajectories(300_000, T, 306).to(DEV)
    huber = torch.nn.HuberLoss(delta=1 / 32, reduction="none")
    rn = osm.RangeNormalizer(shapes=(W, H, T), device=DEV)

    def iteration(cls):
        torch.manual_seed(307)
        sampler = cls(batch_size=512, range_normalizer=rn, dst_range=(-1, 1), fg_trajectories=fg, bg_trajectories=bg,
                      fg_traj_ratio=0.5, num_frames=4)
        m.zero_grad()
        sample = sampler()
        labels = sample["t2_points_normalized"][:, :-1]
        inputs = (sample["t1_points"], sample["source_frame_indices"], sample["target_frame_indices"], sample["frames_set_t"])
        loss = huber(m(inputs), labels).mean()
        emb, fs = m.frame_embeddings, inputs[-1]
        ref_l = c.get_refined_bb_contrastive_loss(tr, m, fs, emb, batch_size=cfg["cl_n_frames"],
                                                  points_per_pair=cfg["cl_points_per_pair"],
                                                  fg_points_ratio=cfg["cl_fg_points_ratio"], temp=cfg["cl_temp"],
                                                  cl_div=cfg["cl_div_ref_bb"])
        dino_l = c.get_dino_bb_contrastive_loss(tr, m, fs)
        raw = m.raw_embeddings
        norm_reg = (emb.norm(dim=1) / raw.norm(dim=1) - 1).abs().mean()
        angle_reg = (torch.einsum("bchw,bchw->bhw", emb, raw) / (emb.norm(dim=1) * raw.norm(dim=1)) - 1).abs().mean()
        loss = loss + cfg["lambda_cl_ref_bb"] * ref_l + cfg["lambda_cl_dino_bb"] * dino_l + \
            cfg["lambda_emb_norm"] * norm_reg + cfg["lambda_angle"] * angle_reg
        loss.backward()
        grads = {k: p.grad.detach().clone() for k, p in list(m.delta_dino.named_parameters()) +
                 [("head." + k, p) for k, p in m.tracker_head.named_parameters()]}
        return sample, loss.detach(), ref_l.detach(), dino_l.detach(), grads

    lib = iteration(sm.DinoTrackerSampler)
    ref = iteration(osm.DinoTrackerSampler)
    again = iteration(osm.DinoTrackerSampler)
    assert_same([lib[0]], [ref[0]])
    assert ref[2].item() != 0.0 and ref[3].item() != 0.0, "both contrastive terms must be active"
    for a, b in zip(lib[1:4], ref[1:4]):
        assert torch.equal(a, b), (a.item(), b.item())
    assert set(lib[4]) == set(ref[4])

    scale = max(v.abs().max().item() for v in ref[4].values())

    def worst(a, b):   # per tensor, against its largest entry (floored at 1e-3 of the largest gradient: the biases ahead
        # of train-mode BatchNorm have gradients that are rounding noise)
        return max((a[k] - b[k]).abs().max().item() / max(b[k].abs().max().item(), 1e-3 * scale) for k in b)
    w_lib, w_run = worst(lib[4], ref[4]), worst(again[4], ref[4])
    print(f"iteration: parameter gradients, library vs oracle sampler {w_lib:.2e}, oracle sampler run twice {w_run:.2e} "
          "(of each tensor's largest entry)")
    assert w_lib <= ITER_GRAD_SPREAD
