"""GPU: the exact-window head (xw_head_kernel, csrc/xwin.cu) -- exact arg-max, 15 x 15 window, refiner, softmax sums and
certificate of two maps per warp -- on the cases its layout has to get right: windows on every border and corner of the
token grid, cells of one map and partial last cells, maps the plan queued next to maps the head finishes or the
certificate queues, and an odd number of maps (a half-empty last pair).  Each is checked against the full-map pipeline,
and four seeded cases against the digest of their anchors as the head computed them before it was fused (one warp per
map, two kernels)."""
import hashlib

import pytest
import torch

from oracle import synth
from oracle.tracker import Geometry

from test_xwin_gpu import _agree, _run

pytestmark = pytest.mark.gpu


def _corner_queries(geo, T):
    """Points on every border and corner of the frame (and one inside), each in a different query frame."""
    xs, ys = (0.0, geo.W / 2, geo.W - 1.0), (0.0, geo.H / 2, geo.H - 1.0)
    pts = [(x, y) for y in ys for x in xs]
    return torch.tensor([[x, y, float(i % T)] for i, (x, y) in enumerate(pts)], dtype=torch.float32)


@pytest.mark.parametrize("kind", ["sharp", "well"])
def test_border_and_corner_windows(kind):
    geo = Geometry(H=140, W=182)            # 19 x 25 tokens: every window near a query touches a border
    T, C = 7, 64                            # 9 queries x 7 frames: an odd number of maps per chunk
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=21, noise=0.15, max_shift=2)
    head = synth.head_weights(kind, seed=21)
    q = _corner_queries(geo, T)
    full, _ = _run(feats, head, q, geo, 0)
    for chunk in (None, 63):
        xw, st = _run(feats, head, q, geo, 1, chunk=chunk)
        _agree(xw, full)
        assert st["pipeline"] == "exact-window" and st["exact_window"] > 0, st


def test_one_map_cells_and_partial_last_cell():
    """T = 129: each (query, anchor frame) pair splits into a cell of 128 maps and a cell of one."""
    geo = Geometry(H=98, W=126)
    T, C = 129, 32
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=8, noise=0.15, max_shift=2)
    head = synth.head_weights("sharp", seed=8)
    q = synth.lattice_query_points(2, 2, geo.H, geo.W, t_q=[0, 50, 100, 128], margin=20.0, jitter_seed=8)
    full, _ = _run(feats, head, q, geo, 0)
    for chunk in (4096, 1001):
        xw, st = _run(feats, head, q, geo, 1, chunk=chunk)
        _agree(xw, full)
        assert st["exact_window"] > 0, st


def test_queued_and_finished_maps_interleaved():
    """A noise frame and a duplicated token make the plan queue maps; they land in the same pairs as maps the head
    finishes."""
    geo = Geometry(H=140, W=182)
    T, C = 6, 64
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=31, noise=0.1, max_shift=1)
    feats[2, :, 3, 4] = feats[2, :, 12, 20]
    feats[3] = synth.random_features(1, C, geo.h, geo.w, seed=32)[0]
    head = synth.head_weights("well", seed=31)
    q = synth.lattice_query_points(4, 3, geo.H, geo.W, t_q=[0, 1, 2, 4] * 3, margin=10.0, jitter_seed=31)
    full, _ = _run(feats, head, q, geo, 0)
    xw, st = _run(feats, head, q, geo, 1)
    print(f"queued and uncertified: {st}")
    _agree(xw, full)
    assert st["pipeline"] == "exact-window" and st["full_map"] > 0, st


def test_exact_window_statistics_match_full_map():
    geo = Geometry()
    T, C = 9, 256
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=16, noise=0.2, max_shift=2)
    head = synth.head_weights("sharp", seed=9)
    q = synth.lattice_query_points(4, 3, geo.H, geo.W, t_q=[i % T for i in range(12)], margin=14.0, jitter_seed=9)
    full, s0 = _run(feats, head, q, geo, 0)
    xw, s1 = _run(feats, head, q, geo, 1)
    _agree(xw, full)
    assert s1["anchor_maps"] == s0["anchor_maps"] == s1["exact_window"] + s1["full_map"]
    assert s1["exact_window"] >= 0.9 * s1["anchor_maps"]


# Anchors digest and "exact-window / full-map / full-map by the certificate" of seeded cases, as the two-kernel head (one
# warp per map, before the fusion) computed them on an H100; the fused head must reproduce every bit.
PINNED = {
    "seeded": ("5f8eb5243c4e2c6d69859fe633169bb31fa73da884381f188b8874f916b9f309", "1380/160/0"),
    "corners_sharp": ("d93090a22f88cb99e5cdb0188307e134eb95b8a33557386965286e23d0166245", "251/36/0"),
    "corners_well": ("2cf32c417de71c82e026d40d665b0b4b37114066a2acae2869d8668b1b2822c7", "121/26/0"),
    "uncertified": ("6baa2b80063ea5e0a8629c257de25058997bbe1e4f84529ef78b9f73bb93c25c", "0/776/658"),
}


def _case(name):
    if name == "seeded":
        geo, T, C, kind, seed, chunk = Geometry(), 10, 128, "sharp", 2024, None
        q = synth.lattice_query_points(5, 4, geo.H, geo.W, t_q=[i % T for i in range(20)], margin=3.0, jitter_seed=2024)
    elif name.startswith("corners"):   # the border path: masked hidden rows and columns, an odd number of maps
        geo, T, C, kind, seed, chunk = Geometry(H=140, W=182), 7, 64, name.split("_")[1], 21, 63
        q = _corner_queries(geo, T)
    else:                              # mixed-sign refiner: the certificate queues most maps, the plan the rest
        geo, T, C, kind, seed, chunk = Geometry(), 8, 64, "mixed", 5, None
        q = synth.lattice_query_points(4, 4, geo.H, geo.W, t_q=[i % T for i in range(16)], margin=10.0, jitter_seed=5)
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=seed, noise=0.2, max_shift=2)
    return feats, synth.head_weights(kind, seed=seed), q, geo, chunk


def case_result(name):
    feats, head, q, geo, chunk = _case(name)
    xw, st = _run(feats, head, q, geo, 1, chunk=chunk)
    digest = hashlib.sha256(xw["anchors"].cpu().numpy().tobytes()).hexdigest()
    return digest, f'{st["exact_window"]}/{st["full_map"]}/{st["full_map_by_certificate"]}', xw


@pytest.mark.parametrize("name", sorted(PINNED))
def test_anchors_bit_identical_to_two_kernel_head(name):
    digest, stats, _ = case_result(name)
    assert (digest, stats) == PINNED[name]


def test_uncertified_maps_queued_and_counted():
    """Maps the certificate queues share pairs with maps the plan queued: the queue branch of the tail and the counter of
    maps queued by the certificate (658 of 776, as the two-kernel head counted them)."""
    digest, stats, xw = case_result("uncertified")
    exact, full_map, by_cert = (int(v) for v in stats.split("/"))
    assert (digest, stats) == PINNED["uncertified"]
    assert full_map > by_cert > 0, stats
    feats, head, q, geo, _ = _case("uncertified")
    full, _ = _run(feats, head, q, geo, 0)
    _agree(xw, full)
