"""CPU checks of the inputs that tests/test_fp16_range_gpu.py feeds the kernels: the oracle is bit-invariant under the
power-of-two scalings used there, and the twin-peak videos have the float64 gaps they were built for.  A failing GPU test
of that file is then about the kernels, not about its inputs."""
import torch

XW_EPS = 1.1e-3    # csrc/xwin.cuh: bound on |coarse - exact| in cosine units
XW_TILE = 128      # tokens per coarse key
XW_SLACK = 3       # a candidate must lie within +-3 tokens of its cell's box centre

from oracle import inference as oi
from oracle import synth
from oracle import tracker as ot
from oracle.tracker import Geometry

SCALES = (-14, -12, -8, 8, 14, 16)   # the exponents of the GPU scale tests
MASSIVE_SCALES = (-4, 2)            # ... and of the massive-activation layout
TWIN_GAPS = (1e-7, 1e-6, 2e-6, 3e-6, 5e-6, 8e-6, 1e-5, 1e-4, 1e-3, 3e-3)   # rungs around the near-tie bound 5e-6
TWIN_SRC, TWIN_DST = (3, 4), (10, 12)   # 13 x 17 tokens: tokens 55 and 182, 8 rows apart, in different 128-token tiles


def test_oracle_is_bit_invariant_under_power_of_two_scaling():
    geo = Geometry(H=98, W=126)
    T, C = 4, 64
    feats, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=11, noise=0.2, max_shift=2)
    head = synth.head_weights("sharp", seed=11)
    q = synth.lattice_query_points(3, 2, geo.H, geo.W, t_q=[0, 1, 2, 3, 0, 1], margin=14.0, jitter_seed=11)
    for layout, scales in (("scaled", SCALES), ("massive", MASSIVE_SCALES)):
        f = feats if layout == "scaled" else synth.massive_channels(feats, seed=11)
        ref = oi.infer(f, q, head, geo, 0.7, 0.6, return_all=True)
        for k in scales:
            got = oi.infer(synth.scaled(f, k), q, head, geo, 0.7, 0.6, return_all=True)
            assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]), (layout, k)
            assert torch.equal(got[2]["cos_sims"], ref[2]["cos_sims"]), (layout, k)
            for n in ref[2]["anchors"]:
                assert torch.equal(got[2]["anchors"][n], ref[2]["anchors"][n]), (layout, k, n)


def test_massive_channels_are_exact_powers_of_two():
    feats = synth.random_features(2, 64, 5, 6, seed=3)
    m = synth.massive_channels(feats, seed=3)
    ratio = (m / feats).reshape(2, 64, -1)[0, :, 0]
    e = torch.log2(ratio.double())
    assert torch.equal(e, e.round())
    assert int((e >= 8).sum()) == 4 and int((e == -6).sum()) == 60


def twin_video(T=len(TWIN_GAPS) + 1, C=128, seed=21):
    geo = Geometry(H=98, W=126)
    base, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=seed, noise=0.05, max_shift=0)
    return geo, synth.twin_peak(base, TWIN_SRC, TWIN_DST, TWIN_GAPS, seed=seed)


def test_twin_peaks_have_the_designed_gaps():
    """For descriptors sampled anywhere inside the source neighbourhood, in any frame: the copy's float64 cosine is the
    original's times (1 - gap) -- measured on the fp32 video the kernels get."""
    geo, feats = twin_video()
    T, C = feats.shape[:2]
    rs = torch.Generator().manual_seed(5)
    for i in range(T):
        off = torch.rand(8, 2, generator=rs) * 2 - 1
        px = geo.patch // 2 + geo.stride * (torch.tensor([TWIN_SRC[1], TWIN_SRC[0]]) + off)
        pts = torch.cat([px, torch.full((8, 1), float(i))], 1)
        d = ot.sample_descriptors(feats.double(), ot.normalize_points_for_sampling(pts, geo)).double()
        for t, gap in enumerate(TWIN_GAPS):
            o = feats[t, :, TWIN_SRC[0], TWIN_SRC[1]].double()
            c = feats[t, :, TWIN_DST[0], TWIN_DST[1]].double()
            co = d @ o / (d.norm(dim=1) * o.norm())
            cc = d @ c / (d.norm(dim=1) * c.norm())
            rel = 1 - cc / co
            assert ((rel - gap).abs() <= 3e-8 + 2e-3 * gap).all(), (i, t, gap, rel)


# Rounding-aligned twins: rn_fp16 orders them against their exact order (synth.rounding_aligned_twin).  NEAR: 3 columns
# apart, in another 128-token tile (tokens 126 / 129), so both are coarse candidates that fit one exact-window box.  FAR: 8
# rows apart (tokens 37 / 183): the candidates leave the box, the map goes to the full-map pipeline.
RA_GAP = 6e-4
RA_NEAR, RA_FAR = ((7, 7), (7, 10)), ((2, 3), (10, 13))


def ra_video(which, T=4, C=128, seed=23):
    geo = Geometry(H=98, W=126)
    base, _ = synth.shifted_field_features(T, C, geo.h, geo.w, seed=seed, noise=0.05, max_shift=0)
    (src, dst) = RA_NEAR if which == "near" else RA_FAR
    feats, gap = synth.rounding_aligned_twin(base, src, dst, RA_GAP, seed=seed)
    return geo, feats, src, dst, gap


def coarse_and_exact(feats, d, frame):
    """Single-pass fp16 cosines (rn_fp16 of both operands, float64 sums, exact norms: the coarse epilogue's quantity) and the
    float64 cosines of descriptor d against every token of `frame`."""
    f = feats[frame].double().reshape(feats.shape[1], -1)
    fh = feats[frame].half().double().reshape(feats.shape[1], -1)
    dd, dh = d.double(), d.half().double()
    den = dd.norm() * f.norm(dim=0)
    return (dh @ fh) / den, (dd @ f) / den


def test_rounding_aligned_twins_reverse_the_coarse_order():
    for which in ("near", "far"):
        geo, feats, src, dst, gap = ra_video(which)
        i_src, i_dst = src[0] * geo.w + src[1], dst[0] * geo.w + dst[1]
        assert i_src // XW_TILE != i_dst // XW_TILE
        near = abs(src[0] - dst[0]) <= XW_SLACK and abs(src[1] - dst[1]) <= XW_SLACK
        assert near == (which == "near")
        o, c = feats[0, :, src[0], src[1]], feats[0, :, dst[0], dst[1]]
        assert (o.half().float().abs() < o.abs()).all() and (c.half().float().abs() > c.abs()).all()   # rounding directions
        T = feats.shape[0]
        px = torch.tensor([geo.patch // 2 + geo.stride * src[1], geo.patch // 2 + geo.stride * src[0]], dtype=torch.float32)
        for i in range(T):   # the descriptor the anchor phase samples at the source token's centre in frame i
            d = ot.sample_descriptors(feats, ot.normalize_points_for_sampling(torch.cat([px, torch.tensor([float(i)])])[None],
                                                                              geo))[0]
            assert torch.equal(d.half(), o.half())
            for a in range(T):
                coarse, exact = coarse_and_exact(feats, d, a)
                assert int(exact.argmax()) == i_src and abs(exact[i_src] - exact[i_dst] - gap) < 1e-6
                assert 1e-4 < coarse[i_dst] - coarse[i_src] and coarse[i_dst] >= coarse.max()   # reversed: the copy leads
                assert (coarse - exact).abs().max() <= XW_EPS
