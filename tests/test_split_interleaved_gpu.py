"""GPU: the fp16 split interleaved per 32 channels (dinotrk_split_hilo) and the exact box GEMM that reads it.

  - split_hilo: every element equals the interleave of dinotrk_split_fp16's hi and lo, bit for bit, and the channels
    past C of the last 32-channel block are zero.  C = 64, 72, 768, 1024 and 1040 (72 and 1040 are not multiples of 32).
  - dinotrk_xw_box_gemm with the interleaved split in the feature struct (128-byte token rows) writes exactly the bytes it
    writes from the separate hi / lo halves (64-byte token rows): cells of <= 64 maps (MB = 64) and of 65..128 maps
    (MB = 128), boxes clipped at every side and corner of the token grid, C = 64, 1024 and 1040, a 1274 x 714 frame's grid.
  - the values from the interleaved split are, through the full-map expression, those of the full-map GEMM
    (dinotrk_corr_maps) at the box tokens.
  - dinotrk_corr_maps with the interleaved split (TcMode::F16X3I, 32-channel K blocks, four ring stages) writes the bytes
    it writes from the separate halves (F16X3): trajectory-phase groups of 256 rows, queue-sized groups, sizes off the
    128 / 256 tiles, on CTA pairs and single CTAs, C = 768, 1024 and 1040 (1040: both runs take F16X3).
"""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BOX, COLS = 21, 448
CANARY = -12345.5
SKIP = -(2 ** 31)
GAP = 3   # descriptor rows before and between cells


@pytest.fixture(scope="module")
def lib():
    from dino_tracker_b200 import _lib
    return _lib


def interleave(hi, lo):
    """[rows][C] hi / lo -> [rows][ceil(C / 32)][64] with zero padding (numpy fp16)."""
    rows, C = hi.shape
    nb = -(-C // 32)
    out = np.zeros((rows, nb, 64), np.float16)
    hp = np.zeros((rows, nb * 32), np.float16)
    lp = np.zeros((rows, nb * 32), np.float16)
    hp[:, :C], lp[:, :C] = hi, lo
    out[:, :, :32] = hp.reshape(rows, nb, 32)
    out[:, :, 32:] = lp.reshape(rows, nb, 32)
    return out.reshape(rows, nb * 64)


@pytest.mark.parametrize("C", [64, 72, 768, 1024, 1040])
def test_hilo_is_the_interleaved_split(lib, C):
    g = torch.Generator(device=DEV).manual_seed(C)
    rows = 777
    x = torch.randn(rows, C, device=DEV, generator=g) * torch.logspace(-3, 3, C, device=DEV)
    x[5] = 0.0
    x[7, :4] = torch.tensor([65504.0, -1e-7, 3e-5, 2.0 ** -24], device=DEV)
    st = lib.stream_ptr()
    hi, lo = lib.split_fp16(x, st)
    hilo = lib.split_hilo(x, st)
    torch.cuda.synchronize()
    assert hilo.shape == (rows, 64 * (-(-C // 32))) and hilo.dtype == torch.float16
    ref = interleave(hi.cpu().numpy(), lo.cpu().numpy())
    assert np.array_equal(hilo.cpu().numpy().view(np.uint16), ref.view(np.uint16))


def test_hilo_batched_shape(lib):
    """A [T][P][C] video splits row by row: the same bytes as its [T P][C] view."""
    x = torch.randn(3, 50, 1040, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    st = lib.stream_ptr()
    a = lib.split_hilo(x, st)
    b = lib.split_hilo(x.reshape(150, 1040), st)
    torch.cuda.synchronize()
    assert a.shape == (3, 50, 33 * 64)
    assert torch.equal(a.reshape(150, -1).view(torch.int16), b.view(torch.int16))


def origins(h, w):
    """Box origins (first row, first column): inside, over every side and corner, and a skipped cell."""
    return [(h // 2 - 10, w // 2 - 10), (-6, -9), (h - 15, w - 12), (-20, w // 2), (h // 3, -20), (10, w - 1), (h - 1, 3),
            (h // 2, SKIP), (h - 21, w - 21), (-3, w - 18), (h - 4, -2), (0, 0)]


# name: (seed, token grid h x w, frames, C, cell sizes)
CASES = {
    "mb64_c1024": (51, (67, 121), 3, 1024, (50, 1, 64, 50, 33, 50, 50, 50, 50, 64, 50, 2)),
    "mb64_c1040": (52, (67, 121), 3, 1040, (50, 1, 64, 50, 33, 50, 50, 50, 50, 64, 50, 2)),
    "mb128_c1024": (53, (67, 121), 3, 1024, (100, 1, 50, 64, 65, 128, 100, 100, 100, 127, 66, 3)),
    "mb128_c64": (54, (67, 121), 2, 64, (128, 65, 1, 50, 64, 100, 100, 128, 100, 70, 90, 128)),
    "mb128_c1040": (55, (67, 121), 2, 1040, (100, 1, 50, 64, 65, 128, 100, 100, 100, 127, 66, 3)),
    "grid1274x714_mb64": (56, (101, 181), 2, 1024, (50, 50, 64, 50, 50, 50, 50, 50, 50, 50, 50, 50)),
    "grid1274x714_mb128": (57, (101, 181), 2, 768, (100, 128, 65, 100, 100, 100, 100, 100, 100, 100, 100, 100)),
}


class Case:
    def __init__(self, lib, seed, hw, T, C, sizes):
        self.lib, self.hw, self.T, self.C = lib, hw, T, C
        h, w = hw
        rng = np.random.default_rng(seed)
        row0, r = [], GAP
        for m in sizes:
            row0.append(r)
            r += m + GAP
        self.rows = r
        self.row0 = np.array(row0, np.int32)
        self.m = np.array(sizes, np.int32)
        self.frame = np.array([k % T for k in range(len(sizes))], np.int32)
        self.org = np.array(origins(h, w)[:len(sizes)], np.int32)
        self.geom = lib.make_geom(14 + 7 * (h - 1), 14 + 7 * (w - 1))
        assert (self.geom.h, self.geom.w) == (h, w)
        st = lib.stream_ptr()
        self.feats = torch.from_numpy(rng.standard_normal((T, h * w, C), dtype=np.float32)).to(DEV)
        self.norms = self.feats.norm(dim=2).contiguous()
        self.f_hi, self.f_lo = lib.split_fp16(self.feats, st)
        self.f_hilo = lib.split_hilo(self.feats, st)
        self.desc = torch.from_numpy(rng.standard_normal((r, C), dtype=np.float32)).to(DEV)
        self.dn = self.desc.norm(dim=1).contiguous()
        self.d_hi, self.d_lo = lib.split_fp16(self.desc, st)
        torch.cuda.synchronize()

    def box(self, hilo):
        lib = self.lib
        fs = lib.make_features(self.feats, self.norms, self.f_hi, self.f_lo, hilo=self.f_hilo if hilo else None)
        xbox = torch.full((self.rows, COLS), CANARY, dtype=torch.float32, device=DEV)
        row0, m, frame = (torch.from_numpy(a).to(DEV) for a in (self.row0, self.m, self.frame))
        org = torch.from_numpy(self.org).to(DEV).contiguous()
        lib.check(lib.load().dinotrk_xw_box_gemm(ctypes.byref(fs), ctypes.byref(self.geom), lib.ptr(self.d_hi),
                                                 lib.ptr(self.d_lo), self.rows, lib.ptr(row0), lib.ptr(m), lib.ptr(frame),
                                                 lib.ptr(org), len(self.m), int(self.m.max()), lib.ptr(xbox),
                                                 lib.stream_ptr()), "xw_box_gemm")
        torch.cuda.synchronize()
        return xbox.cpu().numpy()

    def full_maps(self, f):
        lib, l = self.lib, self.lib.load()
        fs = lib.make_features(self.feats, self.norms, self.f_hi, self.f_lo)
        grp = torch.tensor([[f], [0], [self.rows], [0]], dtype=torch.int32, device=DEV)
        maps = torch.zeros(self.rows, l.dinotrk_map_stride(ctypes.byref(self.geom)), device=DEV)
        nb = l.dinotrk_corr_maps_workspace_bytes(self.rows, 1, self.C)
        ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
        lib.check(l.dinotrk_corr_maps(ctypes.byref(fs), ctypes.byref(self.geom), lib.ptr(self.desc), lib.ptr(self.dn),
                                      lib.ptr(grp[0]), lib.ptr(grp[1]), lib.ptr(grp[2]), lib.ptr(grp[3]), 1, self.rows,
                                      self.rows, lib.ptr(maps), lib.ptr(ws), nb, lib.stream_ptr()), "corr_maps")
        torch.cuda.synchronize()
        return maps.cpu().numpy()

    def box_tokens(self, k):
        h, w = self.hw
        oy, ox = self.org[k]
        by, bx = np.meshgrid(np.arange(BOX), np.arange(BOX), indexing="ij")
        r, c = (oy + by).ravel(), (ox + bx).ravel()
        inside = (r >= 0) & (r < h) & (c >= 0) & (c < w)
        return np.where(inside, r * w + c, 0), inside


@pytest.fixture(scope="module", params=sorted(CASES))
def case(request, lib):
    cs = Case(lib, *CASES[request.param])
    return cs, cs.box(hilo=False), cs.box(hilo=True)


def test_box_gemm_hilo_bit_identical(case):
    cs, ref, got = case
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), \
        f"{int((got.view(np.uint32) != ref.view(np.uint32)).sum())} words differ between the two token-row layouts"
    # the layouts agree on something: computed cells, zero fill outside the grid, untouched canaries
    written = np.zeros(cs.rows, bool)
    for k, (r0, m) in enumerate(zip(cs.row0, cs.m)):
        if cs.org[k][1] != SKIP:
            written[r0:r0 + m] = True
            _, inside = cs.box_tokens(k)
            assert (got[r0:r0 + m, :BOX * BOX][:, ~inside] == 0.0).all()
            assert (got[r0:r0 + m, :BOX * BOX][:, inside] != 0.0).any()
    assert (got[~written] == CANARY).all() and (got[written][:, BOX * BOX:] == CANARY).all()


def test_box_gemm_hilo_matches_full_map_gemm(case):
    cs, _, got = case
    fn = cs.norms.cpu().numpy()
    dn = cs.dn.cpu().numpy()
    for f in sorted(set(cs.frame.tolist())):
        maps = cs.full_maps(f)
        for k, (r0, m) in enumerate(zip(cs.row0, cs.m)):
            if cs.frame[k] != f or cs.org[k][1] == SKIP:
                continue
            tok, inside = cs.box_tokens(k)
            den = np.maximum(dn[r0:r0 + m, None] * fn[f][tok[inside]][None, :], np.float32(1e-8))
            v = np.maximum(got[r0:r0 + m, :BOX * BOX][:, inside] / den, np.float32(0.0))
            ref = maps[r0:r0 + m][:, tok[inside]]
            assert np.array_equal(v, ref), f"cell {k} (m = {m}): {int((v != ref).sum())} values differ from the full map"


# ---- full-map GEMM (dinotrk_corr_maps): TcMode::F16X3I on the interleaved split against F16X3 on the separate halves.
# name: (seed, C, group sizes); the largest group decides the M tile: > 128 rows -> CTA pairs, else single-CTA tiles
CORR_CASES = {
    "pairs_traj_c1024": (61, 1024, (256, 256, 256, 256)),
    "pairs_ragged_c1024": (62, 1024, (300, 1, 129, 513, 9, 255, 257, 40)),
    "single_queue_c1024": (63, 1024, (1, 9, 17, 50, 64, 100, 127, 128, 3, 33)),
    "pairs_c768": (64, 768, (200, 77, 384, 12)),
    "single_c768": (65, 768, (128, 10, 99, 65)),
    "pairs_c1040": (66, 1040, (260, 50, 131)),
    "single_c1040": (67, 1040, (100, 20, 128)),
}


@pytest.mark.parametrize("name", sorted(CORR_CASES))
def test_corr_maps_hilo_byte_identical(lib, name):
    seed, C, sizes = CORR_CASES[name]
    l = lib.load()
    h, w, T = 67, 121, 3
    geom = lib.make_geom(14 + 7 * (h - 1), 14 + 7 * (w - 1))
    g = torch.Generator(device=DEV).manual_seed(seed)
    feats = torch.randn(T, h * w, C, device=DEV, generator=g)
    norms = feats.norm(dim=2).contiguous()
    st = lib.stream_ptr()
    f_hi, f_lo = lib.split_fp16(feats, st)
    f_hilo = lib.split_hilo(feats, st)
    rows = sum(sizes)
    desc = torch.randn(rows, C, device=DEV, generator=g)
    dn = desc.norm(dim=1).contiguous()
    row0 = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int32)
    # groups in a shuffled map order: map0 differs from row0
    order = np.random.default_rng(seed).permutation(len(sizes))
    map0 = np.zeros(len(sizes), np.int32)
    map0[order] = np.concatenate([[0], np.cumsum(np.array(sizes)[order])[:-1]])
    grp = torch.tensor(np.stack([np.arange(len(sizes)) % T, row0, np.array(sizes, np.int32), map0]), dtype=torch.int32,
                       device=DEV).contiguous()
    stride = l.dinotrk_map_stride(ctypes.byref(geom))
    nb = l.dinotrk_corr_maps_workspace_bytes(rows, len(sizes), C)
    out = []
    for hilo in (None, f_hilo):
        fs = lib.make_features(feats, norms, f_hi, f_lo, hilo=hilo)
        maps = torch.full((rows, stride), CANARY, device=DEV)
        ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
        lib.check(l.dinotrk_corr_maps(ctypes.byref(fs), ctypes.byref(geom), lib.ptr(desc), lib.ptr(dn), lib.ptr(grp[0]),
                                      lib.ptr(grp[1]), lib.ptr(grp[2]), lib.ptr(grp[3]), len(sizes), rows, max(sizes),
                                      lib.ptr(maps), lib.ptr(ws), nb, st), "corr_maps")
        torch.cuda.synchronize()
        out.append(maps.cpu().numpy())
    assert (out[0][:, :h * w] > 0).any()
    assert np.array_equal(out[1].view(np.uint32), out[0].view(np.uint32)), \
        f"{int((out[1].view(np.uint32) != out[0].view(np.uint32)).sum())} map words differ"
