"""GPU: the exact box GEMM over many cells per CTA (csrc/xwin.cu, dinotrk_xw_box_gemm_ext).

Each consumer warpgroup loads a cell's description one cell ahead and stages its accumulators through shared memory
before storing them.  With more cells than SMs every CTA runs several cells, so both matter.  One call over 400 cells
(every third skipped, 1 to 64 maps, every extent shape, boxes on and over the border) must store the same bits as one
call per cell, and leave every value outside the extents at its NaN sentinel.
"""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BOX, COLS = 21, 448
SKIP = -(2 ** 31)
HW = (67, 121)
T = 3
N_CELLS = 400
SIZES = (50, 1, 64, 17, 33)


@pytest.mark.parametrize("layout", ["split", "hilo"])
@pytest.mark.parametrize("C", [1024, 72])
def test_many_cells_per_cta_match_one_cell_calls(C, layout):
    from dino_tracker_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(77 + C)
    h, w = HW
    geom = _lib.make_geom(14 + 7 * (h - 1), 14 + 7 * (w - 1))
    st = _lib.stream_ptr()
    feats = torch.from_numpy(rng.standard_normal((T, h * w, C), dtype=np.float32)).to(DEV)
    norms = feats.norm(dim=2).contiguous()
    f_hi, f_lo = _lib.split_fp16(feats, st)
    hilo = _lib.split_hilo(feats, st) if layout == "hilo" else None
    fs = _lib.make_features(feats, norms, f_hi, f_lo, hilo=hilo)
    row0, m, frame, org, ext, r = [], [], [], [], [], 0
    for k in range(N_CELLS):
        mk = SIZES[k % len(SIZES)]
        bh, bw = int(rng.integers(15, BOX + 1)), int(rng.integers(15, BOX + 1))
        row0.append(r)
        m.append(mk)
        r += mk + 1
        frame.append(k % T)
        org.append((int(rng.integers(-6, h - 15)), int(rng.integers(-6, w - 15)) if k % 3 != 1 else SKIP))
        ext.append((int(rng.integers(0, BOX - bh + 1)), int(rng.integers(0, BOX - bw + 1)), bh, bw))
    desc = torch.from_numpy(rng.standard_normal((r, C), dtype=np.float32)).to(DEV)
    d_hi, d_lo = _lib.split_fp16(desc, st)
    cells = {k: torch.tensor(v, dtype=torch.int32, device=DEV).contiguous()
             for k, v in (("row0", row0), ("m", m), ("frame", frame), ("org", org), ("ext", ext))}

    def gemm(out, first, n):
        def at(key):
            t = cells[key]
            return t.data_ptr() + first * t[0].numel() * 4 if t.dim() > 1 else t.data_ptr() + first * 4
        _lib.check(lib.dinotrk_xw_box_gemm_ext(ctypes.byref(fs), ctypes.byref(geom), _lib.ptr(d_hi), _lib.ptr(d_lo), r,
                                               ctypes.c_void_p(at("row0")), ctypes.c_void_p(at("m")),
                                               ctypes.c_void_p(at("frame")), ctypes.c_void_p(at("org")),
                                               ctypes.c_void_p(at("ext")), n, max(SIZES), _lib.ptr(out), st),
                   "xw_box_gemm_ext")

    together = torch.full((r, COLS), float("nan"), dtype=torch.float32, device=DEV)
    alone = torch.full((r, COLS), float("nan"), dtype=torch.float32, device=DEV)
    gemm(together, 0, N_CELLS)
    for k in range(N_CELLS):
        gemm(alone, k, 1)
    torch.cuda.synchronize()
    got, want = together.cpu().numpy().view(np.uint32), alone.cpu().numpy().view(np.uint32)
    written = ~np.isnan(alone.cpu().numpy())
    n_written = sum(m[k] * ext[k][2] * ext[k][3] for k in range(N_CELLS) if org[k][1] != SKIP)
    assert int(written.sum()) == n_written, "the one-cell calls did not write exactly the extents"
    bad = got != want
    assert not bad.any(), f"{int(bad.sum())} values differ between one call and one call per cell"
