"""GPU: the exact box GEMM on each cell's tight extent (csrc/xwin.cu, dinotrk_xw_box_gemm_ext).

The exact-window plan gives each cell an extent inside its 21 x 21 box: the union of its maps' 15 x 15 candidate windows,
15..21 rows by 15..21 columns.  The GEMM lands and multiplies only those tokens.  Checked against the same GEMM on the
whole box (dinotrk_xw_box_gemm), which test_xw_box_gemm_gpu.py holds to the full-map GEMM bit for bit:
  - every extent value is bit-identical to the whole-box run (same operand bytes, same K order of products);
  - every other value of the output (other box columns, columns 441..447, rows between cells, skipped cells) keeps its
    NaN sentinel.
Every (rows, columns) in [15, 21]^2, each at one offset inside the box, with boxes inside the grid, on its edges and
partly or almost wholly outside it; cells of <= 64 maps (one 64-row tile) and of up to 128 (two halves, the parts run one
after the other); C = 1024, 768 and 72 (not a multiple of 32); token rows as separate hi / lo halves and interleaved.
"""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BOX, COLS = 21, 448
SKIP = -(2 ** 31)
GAP = 2   # descriptor rows before and between cells: never written
HW = (67, 121)
T = 3
SIZES = {64: (50, 1, 64, 33), 128: (100, 1, 65, 128, 64)}   # cell sizes, in turn, by the call's largest cell


def origins(h, w):
    """Box origins (first row, first column), in turn: inside, on every edge, over every side and corner, nearly outside."""
    return [(30, 50), (0, 0), (h - BOX, w - BOX), (-6, -9), (h - 15, w - 12), (20, -20), (-20, 60), (10, w - 1), (h - 1, 3),
            (0, 40), (33, w - BOX), (h - BOX, 0)]


def make_case(seed, C, mb):
    rng = np.random.default_rng(seed)
    h, w = HW
    feats = rng.standard_normal((T, h * w, C), dtype=np.float32)
    exts = [(bh, bw) for bh in range(15, BOX + 1) for bw in range(15, BOX + 1)]
    org = origins(h, w)
    sizes = SIZES[mb]
    row0, m, frame, box_org, box_ext, r = [], [], [], [], [], GAP
    for k, (bh, bw) in enumerate(exts + [(15, 15)]):
        mk = sizes[k % len(sizes)]
        row0.append(r)
        m.append(mk)
        r += mk + GAP
        frame.append(k % T)
        box_org.append(org[k % len(org)] if k < len(exts) else (25, SKIP))   # the last cell is skipped
        box_ext.append((int(rng.integers(0, BOX - bh + 1)), int(rng.integers(0, BOX - bw + 1)), bh, bw))
    desc = rng.standard_normal((r, C), dtype=np.float32)
    return dict(feats=feats, desc=desc, C=C, row0=np.array(row0, np.int32), m=np.array(m, np.int32),
                frame=np.array(frame, np.int32), org=np.array(box_org, np.int32), ext=np.array(box_ext, np.int32))


def run(cs, layout):
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    h, w = HW
    geom = _lib.make_geom(14 + 7 * (h - 1), 14 + 7 * (w - 1))
    st = _lib.stream_ptr()
    feats = torch.from_numpy(cs["feats"]).to(DEV)
    norms = feats.norm(dim=2).contiguous()
    f_hi, f_lo = _lib.split_fp16(feats, st)
    hilo = _lib.split_hilo(feats, st) if layout == "hilo" else None
    fs = _lib.make_features(feats, norms, f_hi, f_lo, hilo=hilo)
    desc = torch.from_numpy(cs["desc"]).to(DEV)
    d_hi, d_lo = _lib.split_fp16(desc, st)
    rows = desc.shape[0]
    row0, m, frame, org, ext = (torch.from_numpy(cs[k]).to(DEV).contiguous() for k in ("row0", "m", "frame", "org", "ext"))
    n, max_m = len(cs["m"]), int(cs["m"].max())
    whole = torch.full((rows, COLS), float("nan"), dtype=torch.float32, device=DEV)
    tight = torch.full((rows, COLS), float("nan"), dtype=torch.float32, device=DEV)
    _lib.check(lib.dinotrk_xw_box_gemm(ctypes.byref(fs), ctypes.byref(geom), _lib.ptr(d_hi), _lib.ptr(d_lo), rows, _lib.ptr(row0),
                                       _lib.ptr(m), _lib.ptr(frame), _lib.ptr(org), n, max_m, _lib.ptr(whole), st), "xw_box_gemm")
    _lib.check(lib.dinotrk_xw_box_gemm_ext(ctypes.byref(fs), ctypes.byref(geom), _lib.ptr(d_hi), _lib.ptr(d_lo), rows,
                                           _lib.ptr(row0), _lib.ptr(m), _lib.ptr(frame), _lib.ptr(org), _lib.ptr(ext), n, max_m,
                                           _lib.ptr(tight), st), "xw_box_gemm_ext")
    torch.cuda.synchronize()
    return whole.cpu().numpy(), tight.cpu().numpy()


@pytest.mark.parametrize("layout", ["split", "hilo"])
@pytest.mark.parametrize("mb", [64, 128])
@pytest.mark.parametrize("C", [1024, 768, 72])
def test_tight_extent_bit_identical_to_whole_box(C, mb, layout):
    cs = make_case(1000 + C + mb, C, mb)
    whole, tight = run(cs, layout)
    nan_bits = np.float32("nan").view(np.uint32)
    expect = np.full(tight.shape, nan_bits, np.uint32)
    n_cells = 0
    for k, (r0, mk) in enumerate(zip(cs["row0"], cs["m"])):
        if cs["org"][k][1] == SKIP:
            continue
        y, x, bh, bw = cs["ext"][k]
        cols = ((y + np.arange(bh))[:, None] * BOX + x + np.arange(bw)[None, :]).ravel()
        assert not np.isnan(whole[r0:r0 + mk][:, cols]).any(), f"cell {k}: the whole-box run left an extent value unwritten"
        expect[r0:r0 + mk, cols] = whole[r0:r0 + mk][:, cols].view(np.uint32)
        n_cells += 1
    assert n_cells == 49
    got = tight.view(np.uint32)
    bad = got != expect
    if bad.any():
        rr, cc = np.nonzero(bad)
        k = int(np.searchsorted(cs["row0"], rr[0], side="right") - 1)
        raise AssertionError(f"{int(bad.sum())} values differ; first at row {rr[0]} column {cc[0]} (cell {k}, extent "
                             f"{cs['ext'][k].tolist()}, origin {cs['org'][k].tolist()}): {tight[rr[0], cc[0]]!r} vs "
                             f"{expect[rr[0], cc[0]].view(np.float32)!r}")
