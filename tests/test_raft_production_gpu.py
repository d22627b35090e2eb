"""GPU suite: RAFT-large (dino_tracker_b200/raft.py, csrc/raft.cu) where tests/test_raft_gpu.py does not reach:

  - the update block's row chunks: a call of P pairs runs every convolution on M = P * h8 * w8 rows in passes of
    RAFT_ROWS rows, and from the second pass on the epilogue rows, the row scales and the in-place GRU and flow updates
    are offset into the call; production calls (trajectories.video_flows at 480 x 856) take 8 and more passes;
  - frame sizes whose padding to a multiple of 8 is uneven (the "sintel" split puts the smaller half on top / left);
  - the encoders on their own against float64, on textured frames and on flat ones (InstanceNorm variance near zero);
  - pair lists with self pairs, repeats, other orders, and a memory budget that splits them unevenly;
  - dinotrk_raft_flow's check that every flow starts from a frame encoded with its context.

Flow bars are those of tests/test_raft_gpu.py: against torchvision in float64, at most FP32_BAR x torchvision fp32's own
error (floor 1e-4 px) and at most a tenth of torchvision's TF32 default.  Encoder bar: pinned from the H100 run (numbers
in DESIGN.md 4.8)."""
import contextlib
import ctypes

import pytest
import torch

from oracle import raft as oraft
from test_raft_gpu import DEV, FP32_BAR, pair, padded, tv_flows

pytestmark = pytest.mark.gpu
RAFT_ROWS = 32768       # csrc/raft.cu RAFT_ROWS: rows of one im2col / GEMM pass of the update block
# encoder error (relative to the largest float64 entry) at most this multiple of the fp32 oracle's (measured on an H100
# 80GB HBM3 at 700 W: fmap 1.1x to 1.6x, ctx 3.6x to 6.9x)
ENC_BAR = {"fmap": 4, "ctx": 15}


@pytest.fixture(scope="module")
def model():
    return oraft.seeded_model().to(DEV)


@pytest.fixture(scope="module")
def lib_raft(model):
    from dino_tracker_b200.raft import RaftLarge
    return RaftLarge(model, device=DEV)


def video(T, H, W, step):
    return torch.cat([oraft.textured_pair(H, W, (step[0] * t, step[1] * t))[1] for t in range(T)]).to(DEV)


def chunk_layout(tag, pairs, H, W):
    """M of one flow call and the pairs its RAFT_ROWS pass boundaries fall in (printed)."""
    hw = -(-H // 8) * -(-W // 8)
    M = len(pairs) * hw
    cuts = [(b, b // hw, b % hw) for b in range(RAFT_ROWS, M, RAFT_ROWS)]
    print(f"{tag}: {len(pairs)} pairs x {hw} rows: M = {M}, {len(cuts) + 1} passes; boundaries: "
          + ", ".join(f"row {b} = pair {k} {pairs[k]} row {r}" for b, k, r in cuts))
    return M, cuts


def check_flows(tag, ours, refs, bad):
    """ours [P][2][H][W]; refs: (float64, fp32, fp32 + TF32) torchvision flows of the same pairs.  Appends failures to
    ``bad``; returns the fp32 bar of each pair."""
    ref, f32, tf32 = refs
    bars = []
    for d in range(ours.shape[0]):
        e_lib = (ours[d].double() - ref[d]).abs().max().item()
        e_f32 = (f32[d] - ref[d]).abs().max().item()
        e_tf32 = (tf32[d] - ref[d]).abs().max().item()
        bar = max(FP32_BAR * e_f32, 1e-4)
        print(f"{tag} [{d}]: max|flow|={ref[d].abs().max().item():.3f}  library {e_lib:.3e}  (bar {bar:.3e} = "
              f"max({FP32_BAR} x fp32 {e_f32:.3e}, 1e-4); bar {0.1 * e_tf32:.3e} = 0.1 x fp32+TF32 {e_tf32:.3e})")
        if e_lib > bar or e_lib > 0.1 * e_tf32:
            bad.append((tag, d, e_lib, e_f32, e_tf32))
        bars.append(bar)
    return bars


def tv_refs(model, a, b, ns):
    """[(float64, fp32, fp32 + TF32) torchvision flows of the frame pairs (a[k], b[k])] for each n in ns."""
    runs = [tv_flows(model, a, b, ns, dt, tf32) for dt, tf32 in
            ((torch.float64, False), (torch.float32, False), (torch.float32, True))]
    return list(zip(*runs))


# ---- row chunks --------------------------------------------------------------------------------------------------------

def test_row_chunks_at_476x854_bit_for_bit(model, lib_raft):
    """12 pairs of a 7-frame video (both directions, gaps up to 6 frames) in one call: M = 77,040 rows, three passes
    whose boundaries fall inside pairs 5 and 10.  Every pair has the bits of the same pair run alone (M = 6,420, one
    pass), and the two straddling pairs are within the bars against torchvision float64."""
    T, H, W = 7, 476, 854
    v = video(T, H, W, (1.3, -0.8))
    enc = lib_raft.encode(v)
    assert enc.hi is not None
    pairs = [(0, 1), (1, 0), (0, 6), (6, 0), (2, 4), (4, 2), (5, 3), (3, 5), (1, 5), (5, 1), (6, 2), (2, 6)]
    M, cuts = chunk_layout(f"RAFT {H}x{W}", pairs, H, W)
    assert M > 2 * RAFT_ROWS and lib_raft.batch_pairs(H, W) >= len(pairs)      # one call, three passes
    straddle = [k for _, k, r in cuts if r > 0]
    assert straddle == [5, 10]
    batch = lib_raft.flows(enc, pairs, 24)
    for k, p in enumerate(pairs):
        assert torch.equal(batch[k], lib_raft.flows(enc, [p], 24)[0]), p
    a = torch.stack([v[pairs[k][0]] for k in straddle])
    b = torch.stack([v[pairs[k][1]] for k in straddle])
    bad = []
    check_flows(f"RAFT {H}x{W} straddling pairs {[pairs[k] for k in straddle]} n=24", batch[straddle],
                tv_refs(model, a, b, (24,))[0], bad)
    assert not bad, bad


def test_row_chunks_all_pairs_of_9_frames_at_136x248(lib_raft):
    """All 72 ordered pairs of a 9-frame video in one call (M = 37,944 rows, two passes) against 72 single-pair calls."""
    T, H, W = 9, 136, 248
    enc = lib_raft.encode(video(T, H, W, (0.7, -0.4)))
    pairs = [(i, j) for i in range(T) for j in range(T) if i != j]
    M, cuts = chunk_layout(f"RAFT {H}x{W}", pairs, H, W)
    assert M > RAFT_ROWS and cuts[0][2] > 0
    batch = lib_raft.flows(enc, pairs, 12)
    for k, p in enumerate(pairs):
        assert torch.equal(batch[k], lib_raft.flows(enc, [p], 12)[0]), p


def test_video_flows_route_at_476x854(lib_raft):
    """trajectories.video_flows with the direct filter on a 10-frame video: the consecutive group (18 pairs, M =
    115,560 rows) and the direct groups of start frames 0 (18 pairs) and 8 give the bits of single-pair calls."""
    from dino_tracker_b200.trajectories import video_flows
    T, H, W = 10, 476, 854
    v = video(T, H, W, (0.6, 0.35))
    consecutive = [(i, i + 1) for i in range(T - 1)] + [(i + 1, i) for i in range(T - 1)]
    M, _ = chunk_layout(f"RAFT video_flows {H}x{W} consecutive", consecutive, H, W)
    assert M > 3 * RAFT_ROWS and lib_raft.batch_pairs(H, W) >= len(consecutive)
    fwd, bwd, direct = video_flows(v, lib_raft, True, DEV)
    enc = lib_raft.encode(v)

    def one(i, j):
        return lib_raft.flows(enc, [(i, j)])[0]

    for i in range(T - 1):
        assert torch.equal(fwd[i], one(i, i + 1)), i
        assert torch.equal(bwd[i], one(i + 1, i)), i
    for s in range(T - 1):                      # the provider yields the direct groups in start-frame order
        f, b = direct(s)
        assert f.shape[0] == b.shape[0] == T - 1 - s
        if s in (0, T - 2):
            for k in range(T - 1 - s):
                assert torch.equal(f[k], one(s, s + 1 + k)), (s, k)
                assert torch.equal(b[k], one(s + 1 + k, s)), (s, k)


# ---- uneven padding ----------------------------------------------------------------------------------------------------

def off_by_one(f, ref):
    """max |f - ref| of a flow f [2][H][W] moved by one row and by one column, either way: the error of a crop that is off
    by one pixel."""
    d = lambda x, y: (x - y).abs().max().item()
    return (min(d(f[:, 1:], ref[:, :-1]), d(f[:, :-1], ref[:, 1:])),
            min(d(f[:, :, 1:], ref[:, :, :-1]), d(f[:, :, :-1], ref[:, :, 1:])))


@pytest.mark.parametrize("H,W", [(121, 121), (127, 129), (475, 853), (473, 849)])
def test_uneven_padding_against_torchvision_float64(model, lib_raft, H, W):
    """Padding splits 3+4 / 3+4, 0+1 / 3+4, 2+3 / 1+2 and 3+4 / 3+4 (top+bottom / left+right), both directions, n = 1,
    12, 24.  A crop one row or one column off exceeds the bar by at least 100x, so the bar tells the crops apart."""
    _, pad = padded(torch.zeros(1, 3, H, W))
    print(f"RAFT {H}x{W}: padded to {H + pad[2] + pad[3]}x{W + pad[0] + pad[1]}, rows {pad[2]}+{pad[3]}, "
          f"columns {pad[0]}+{pad[1]}")
    a, b = pair(H, W)
    enc = lib_raft.encode(torch.cat([a, b]))
    assert enc.hi is not None
    ns = (1, 12, 24)
    refs = tv_refs(model, torch.cat([a, b]), torch.cat([b, a]), ns)
    bad = []
    for n, r in zip(ns, refs):
        ours = lib_raft.flows(enc, [(0, 1), (1, 0)], n)
        bars = check_flows(f"RAFT {H}x{W} n={n}", ours, r, bad)
        for d in range(2):
            rows, cols = off_by_one(ours[d].double(), r[0][d])
            print(f"RAFT {H}x{W} n={n} [{d}]: one row off {rows:.3e} ({rows / bars[d]:.0f}x the bar), one column off "
                  f"{cols:.3e} ({cols / bars[d]:.0f}x)")
            if min(rows, cols) < 100 * bars[d]:
                bad.append(("crop sensitivity", n, d, rows, cols, bars[d]))
    assert not bad, bad


# ---- encoders ----------------------------------------------------------------------------------------------------------

@contextlib.contextmanager
def no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def encoder_frames(H, W):
    """{name: frame [3][H][W] in [0, 1]}."""
    tex = oraft.textured_pair(H, W)[0][0]
    colour = torch.tensor([0.8, 0.3, 0.1]).view(3, 1, 1)
    box = tex.clone()
    box[:, :H // 8] = 0.0
    box[:, H - H // 8:] = 0.0
    xs = torch.arange(W).view(1, 1, W)
    return {"textured": tex,
            "constant colour": colour.expand(3, H, W),
            # maps to 0 everywhere, padding included: all-zero im2col rows, and every InstanceNorm of the feature
            # encoder sees an exactly constant channel (variance 0, rstd = 1 / sqrt(1e-5))
            "mid grey": torch.full((3, H, W), 0.5),
            "letterbox": box,
            "vertical step": torch.where(xs < W // 2 + 3, colour, 1.0 - colour).expand(3, H, W)}


def oracle_encode(model, frames, dtype):
    """oracle/raft.py's encoders in ``dtype`` (TF32 off) on the sintel-padded frames: fmap, ctx [N][256][h8][w8] in
    float64, ctx = tanh(hidden) | relu(context)."""
    sd = {k: v.to(dtype) for k, v in model.state_dict().items()}
    with no_tf32(), torch.no_grad():
        fmap, hidden, context = oraft.encode(sd, padded(frames)[0].to(dtype))
    return fmap.double(), torch.cat([hidden, context], 1).double()


@pytest.mark.filterwarnings("ignore:RAFT feature maps outside")   # flat frames' fmaps; no flow runs here
@pytest.mark.parametrize("H,W", [(128, 128), (475, 853), (476, 854)])
def test_encoders_against_float64(model, lib_raft, H, W):
    """encode's fmap and ctx against oracle/raft.py's encoders in float64 on the same sintel-padded frames, per frame,
    relative to the largest float64 entry."""
    frames = encoder_frames(H, W)
    x = torch.stack(list(frames.values())).to(DEV)
    enc = lib_raft.encode(x)
    assert bool(torch.isfinite(enc.fmap).all()) and bool(torch.isfinite(enc.ctx).all())
    h8, w8 = -(-H // 8), -(-W // 8)
    lib = [t.view(len(frames), h8, w8, 256).permute(0, 3, 1, 2).double() for t in (enc.fmap, enc.ctx)]
    ref = oracle_encode(model, x, torch.float64)
    f32 = oracle_encode(model, x, torch.float32)
    # Mid grey: each normalised channel is exactly 0, so the fmap is exactly the last convolution's bias.  torch's
    # InstanceNorm can leave the rounding of a constant channel's mean in its output, and each further InstanceNorm
    # multiplies such constants, once the zero padding has made them vary, by up to 1 / sqrt(1e-5): the fp32 oracle's
    # fmap is then rounding noise (off by 21 at 480 x 856 on an H100; float64 on a CPU is off by 11 at 128 x 128), so
    # the exact value is the reference and the fp32 error no bar.
    grey = list(frames).index("mid grey")
    bias = model.state_dict()["feature_encoder.conv.bias"].float()
    noise = [(r[grey] - bias.double().view(256, 1, 1)).abs().max().item() for r in (ref[0], f32[0])]
    print(f"RAFT encoder {H}x{W} mid grey fmap: library == bias {torch.equal(enc.fmap[grey], bias.expand(h8 * w8, 256))}; "
          f"max|oracle - bias| float64 {noise[0]:.3e}, fp32 {noise[1]:.3e} (max|bias| {bias.abs().max().item():.3e})")
    assert torch.equal(enc.fmap[grey], bias.expand(h8 * w8, 256))
    bad = []
    for o, out in enumerate(("fmap", "ctx")):
        scale = ref[o].abs().amax(dim=(1, 2, 3))
        e_lib = ((lib[o] - ref[o]).abs().amax(dim=(1, 2, 3)) / scale).tolist()
        e_f32 = ((f32[o] - ref[o]).abs().amax(dim=(1, 2, 3)) / scale).tolist()
        for k, name in enumerate(frames):
            if out == "fmap" and k == grey:
                continue
            bar = ENC_BAR[out] * e_f32[k]
            print(f"RAFT encoder {H}x{W} {name:15s} {out}: max|x|={scale[k].item():.3f}  library {e_lib[k]:.3e}  "
                  f"oracle fp32 {e_f32[k]:.3e}  (bar {bar:.3e})")
            if e_lib[k] > bar:
                bad.append((out, name, e_lib[k], e_f32[k]))
    assert not bad, bad


# ---- pair lists --------------------------------------------------------------------------------------------------------

def test_self_pairs_against_torchvision_float64(model, lib_raft):
    H, W = 136, 248
    a, b = pair(H, W)
    enc = lib_raft.encode(torch.cat([a, b]))
    ours = lib_raft.flows(enc, [(0, 0), (1, 1)], 12)
    bad = []
    check_flows(f"RAFT {H}x{W} self pairs n=12", ours, tv_refs(model, torch.cat([a, b]), torch.cat([a, b]), (12,))[0],
                bad)
    assert not bad, bad
    mixed = lib_raft.flows(enc, [(0, 1), (1, 1), (1, 0), (0, 0)], 12)
    assert torch.equal(mixed[1], ours[1]) and torch.equal(mixed[3], ours[0])


class _CountingLib:
    """The library with the n_pairs of every dinotrk_raft_flow call recorded."""

    def __init__(self, lib):
        self._l, self.calls = lib, []

    def __getattr__(self, name):
        return getattr(self._l, name)

    def dinotrk_raft_flow(self, *args):
        self.calls.append(args[9])
        return self._l.dinotrk_raft_flow(*args)


def test_pair_lists_repeats_orders_and_an_uneven_budget(lib_raft):
    from dino_tracker_b200.raft import RaftLarge
    T, H, W = 5, 136, 248
    enc = lib_raft.encode(video(T, H, W, (0.7, -0.4)))
    asc = [(i, j) for i in range(T) for j in range(T) if i != j]
    ref = dict(zip(asc, lib_raft.flows(enc, asc, 12)))
    # the same pair twice in one call
    twice = lib_raft.flows(enc, [(0, 1), (3, 2), (0, 1)], 12)
    assert torch.equal(twice[0], twice[2]) and torch.equal(twice[0], ref[(0, 1)])
    # descending, and each pair next to its reverse
    for order in (asc[::-1], [p for i in range(T) for j in range(i + 1, T) for p in ((j, i), (i, j))]):
        f = lib_raft.flows(enc, order, 12)
        for k, p in enumerate(order):
            assert torch.equal(f[k], ref[p]), p
    # a budget of 3 pairs: 7 pairs run as 3 + 3 + 1
    one, two = (lib_raft._lib.dinotrk_raft_flow_workspace_bytes(H, W, n) for n in (1, 2))
    small = RaftLarge.__new__(RaftLarge)
    small.__dict__.update(lib_raft.__dict__)
    small.memory_budget = one + 2 * (two - one)
    small._lib = _CountingLib(lib_raft._lib)
    assert small.batch_pairs(H, W) == 3
    seven = asc[3:10]
    f = small.flows(enc, seven, 12)
    assert small._lib.calls == [3, 3, 1]
    assert torch.equal(f, lib_raft.flows(enc, seven, 12))


# ---- C API -------------------------------------------------------------------------------------------------------------

def test_flow_from_a_frame_without_context_is_refused_before_any_launch(lib_raft):
    """dinotrk_raft_flow with ctx for the first T_ctx frames refuses a pair starting at frame i >= T_ctx (it would read
    past ctx), and T_ctx outside [1, T], before any launch."""
    from dino_tracker_b200 import _lib
    H, W = 128, 128
    enc = lib_raft.encode(torch.cat(pair(H, W)), n_context=1)
    assert enc.T == 2 and enc.ctx.shape[0] == 1
    lib = _lib.load()
    ws = torch.empty(lib.dinotrk_raft_flow_workspace_bytes(H, W, 1), device=DEV, dtype=torch.uint8)
    out = torch.empty(1, 2, H, W, device=DEV)

    def call(i, j, t_ctx):
        with torch.cuda.device(DEV):
            rc = lib.dinotrk_raft_flow(_lib.ptr(enc.fmap), _lib.ptr(enc.hi), _lib.ptr(enc.lo), _lib.ptr(enc.ctx), enc.T,
                                       t_ctx, H, W, (ctypes.c_int * 2)(i, j), 1, 3, ctypes.byref(lib_raft._w),
                                       _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
        _lib.check(rc, "raft_flow")

    for i, j, t_ctx, msg in ((1, 0, 1, "without its context"), (0, 1, 0, "bad arguments"), (0, 1, 3, "bad arguments")):
        before = _lib.launch_count()
        with pytest.raises(_lib.DinotrkError, match=msg):
            call(i, j, t_ctx)
        assert _lib.launch_count() == before, (i, j, t_ctx)
    with pytest.raises(_lib.DinotrkError):
        lib_raft.flows(enc, [(1, 0)])
    before = _lib.launch_count()
    call(0, 1, 1)
    assert _lib.launch_count() > before
    assert torch.equal(out[0], lib_raft.flows(enc, [(0, 1)], 3)[0])
