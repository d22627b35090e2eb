"""RAFT-large optical flow on libdinotrk (include/dinotrk.h: dinotrk_raft_encode / dinotrk_raft_flow).

``RaftLarge`` runs torchvision's ``raft_large`` forward pass (eval mode) with torchvision's weights as they are: built
from a ``raft_large`` module or its ``state_dict`` (so a cached ``Raft_Large_Weights`` checkpoint loads as is; nothing is
downloaded).  Each frame of a video is encoded once; the flows of a list of frame pairs then run as one batch of pairs
(the correlation pyramids and the update loop on pairs x h/8 x w/8 rows), capped by a memory budget.  A pair's flow is
the same bits in any batch.

Three ways in:
  - ``encode(video01)`` / ``flows(enc, pairs, num_flow_updates)``;
  - ``model(a, b)``: the ``flow_fn`` contract of ``trajectories.extract_trajectories`` (frames a, b [B][3][H][W] in
    [0, 1] -> flows a -> b [B][2][H][W]);
  - ``video_flows(video01, groups)``: encodes the video once and yields the flows of each group of pairs, which
    ``extract_trajectories`` / ``preprocess_video`` use for the consecutive and the direct flows.
"""
import ctypes
import warnings

import torch

from . import _lib

# torchvision key prefix of every convolution, in the order of include/dinotrk.h's dinotrk_raft_weights; "zr" entries
# are a GRU's convz and convr stacked
_BLOCKS = [("layer1.0", False), ("layer1.1", False), ("layer2.0", True), ("layer2.1", False), ("layer3.0", True),
           ("layer3.1", False)]


def _encoder_keys(prefix):
    keys = [prefix + "convnormrelu"]
    for blk, ds in _BLOCKS:
        keys += [f"{prefix}{blk}.convnormrelu1", f"{prefix}{blk}.convnormrelu2"] + ([f"{prefix}{blk}.downsample"] if ds else [])
    return keys + [prefix + "conv"]


_UPDATE_KEYS = ["update_block.motion_encoder.convcorr1.0", "update_block.motion_encoder.convcorr2.0",
                "update_block.motion_encoder.convflow1.0", "update_block.motion_encoder.convflow2.0",
                "update_block.motion_encoder.conv.0",
                "update_block.recurrent_block.convgru1.zr", "update_block.recurrent_block.convgru1.convq",
                "update_block.recurrent_block.convgru2.zr", "update_block.recurrent_block.convgru2.convq",
                "update_block.flow_head.conv1", "update_block.flow_head.conv2",
                "mask_predictor.convrelu.0", "mask_predictor.conv"]
CONV_KEYS = _encoder_keys("feature_encoder.") + _encoder_keys("context_encoder.") + _UPDATE_KEYS
assert len(CONV_KEYS) == _lib.RAFT_NCONV


def _np(cout):
    return 64 if cout <= 64 else 128 if cout <= 128 else -(-cout // 256) * 256


def conv_matrices(state_dict):
    """[(weight [Np][Kp] fp32, bias [Np] fp32)] of every convolution in the library's order and layout: K-major
    (ky, kx, ci), zero padded; the context encoder's eval-mode BatchNorm folded in (float64 arithmetic)."""
    sd = {k: v.detach().to("cpu", torch.float64) for k, v in state_dict.items()}
    out = []
    for key in CONV_KEYS:
        if key.endswith(".zr"):
            base = key[:-3]
            w = torch.cat([sd[base + ".convz.weight"], sd[base + ".convr.weight"]])
            b = torch.cat([sd[base + ".convz.bias"], sd[base + ".convr.bias"]])
        elif key + ".weight" in sd:                      # plain Conv2d
            w, b = sd[key + ".weight"], sd[key + ".bias"]
        else:                                            # Conv2dNormActivation: [conv, norm, (relu)]
            w, b = sd[key + ".0.weight"], sd[key + ".0.bias"]
            if key.startswith("context_encoder.") and key + ".1.running_mean" in sd:
                s = sd[key + ".1.weight"] / torch.sqrt(sd[key + ".1.running_var"] + 1e-5)
                w = w * s[:, None, None, None]
                b = (b - sd[key + ".1.running_mean"]) * s + sd[key + ".1.bias"]
        cout = w.shape[0]
        m = w.permute(0, 2, 3, 1).reshape(cout, -1)
        kp, np_ = -(-m.shape[1] // 8) * 8, _np(cout)
        mat = torch.zeros(np_, kp, dtype=torch.float64)
        mat[:cout, :m.shape[1]] = m
        bias = torch.zeros(np_, dtype=torch.float64)
        bias[:cout] = b
        out.append((mat.float(), bias.float()))
    return out


class RaftEncoding:
    """Per-frame encodings of a video: fmap [T][h8 * w8][256], ctx [T][h8 * w8][256], the fmap's fp16 split (None when
    outside its faithful range: the correlation volume then runs on the exact-fp32 GEMM)."""

    def __init__(self, fmap, ctx, hi, lo, H, W):
        self.fmap, self.ctx, self.hi, self.lo, self.H, self.W = fmap, ctx, hi, lo, H, W

    @property
    def T(self):
        return self.fmap.shape[0]


class RaftLarge:
    """torchvision ``raft_large`` (eval mode) on the library.  ``model``: a ``raft_large`` module or its state_dict.
    ``memory_budget``: bytes of workspace one batch of pairs may take (the pyramids are ~219 MB per pair at 480 x 856)."""

    def __init__(self, model, device="cuda:0", num_flow_updates=24, memory_budget=8 << 30):
        self._dev = _lib.require_cuda(device)
        sd = model.state_dict() if isinstance(model, torch.nn.Module) else model
        self.num_flow_updates = int(num_flow_updates)
        self.memory_budget = int(memory_budget)
        self._lib = _lib.load()
        self._tensors = []
        self._w = _lib.RaftWeights()
        with torch.cuda.device(self._dev):
            st = _lib.stream_ptr()
            for i, (mat, bias) in enumerate(conv_matrices(sd)):
                # largest entry into [2^13, 2^14): the lo halves of small weights stay normal fp16 numbers
                e = 14 - int(torch.frexp(mat.abs().max()).exponent) if mat.abs().max() > 0 else 0
                self._w.scale[i] = 2.0 ** -e
                mat, bias = (mat * 2.0 ** e).to(self._dev), bias.to(self._dev)
                hi, lo = _lib.split_fp16(mat, st)
                self._tensors += [hi, lo, bias]
                self._w.w_hi[i], self._w.w_lo[i], self._w.bias[i] = hi.data_ptr(), lo.data_ptr(), bias.data_ptr()

    def _ws(self, nbytes):
        if nbytes == 0:
            raise _lib.DinotrkError("RAFT: invalid frame size (frames must be at least 121 x 121)")
        return torch.empty(nbytes, device=self._dev, dtype=torch.uint8)

    @_lib.on_device
    @torch.no_grad()
    def encode(self, video01, n_context=None):
        """video01 [T][3][H][W] in [0, 1] -> RaftEncoding (one encoding per frame).  Only the first ``n_context`` frames
        (default: all) get the context encoder: flows can start from those only."""
        v = video01.to(self._dev, torch.float32).contiguous()
        T, _, H, W = v.shape
        h8, w8 = -(-H // 8), -(-W // 8)
        n_ctx = T if n_context is None else int(n_context)
        fmap = torch.empty(T, h8 * w8, 256, device=self._dev)
        ctx = torch.empty(n_ctx, h8 * w8, 256, device=self._dev)
        ws = self._ws(self._lib.dinotrk_raft_encode_workspace_bytes(H, W))
        st = _lib.stream_ptr()
        _lib.check(self._lib.dinotrk_raft_encode(_lib.ptr(v), T, n_ctx, H, W, ctypes.byref(self._w), _lib.ptr(fmap),
                                                 _lib.ptr(ctx) if n_ctx else None, _lib.ptr(ws), ws.numel(), st), "raft_encode")
        del ws
        norms = torch.empty(T, h8 * w8, device=self._dev)
        _lib.check(self._lib.dinotrk_token_norms(_lib.ptr(fmap), _lib.ptr(norms), T, 256, h8 * w8, st), "token_norms")
        max_abs, min_norm, ok = _lib.split_range(fmap, norms, st)
        hi = lo = None
        if ok:
            hi, lo = _lib.split_fp16(fmap, st)
        else:
            warnings.warn(f"RAFT feature maps outside the fp16 split's faithful range (max |x| = {max_abs:.3g}, smallest "
                          f"norm = {min_norm:.3g}): the correlation volumes run on the exact-fp32 GEMM", RuntimeWarning,
                          stacklevel=3)
        return RaftEncoding(fmap, ctx, hi, lo, H, W)

    def batch_pairs(self, H, W):
        """Pairs per flow call within the memory budget (at least 1)."""
        one, two = (self._lib.dinotrk_raft_flow_workspace_bytes(H, W, n) for n in (1, 2))
        if one == 0:
            raise _lib.DinotrkError("RAFT: invalid frame size (frames must be at least 121 x 121)")
        per = two - one
        return max(1, (self.memory_budget - (one - per)) // per)

    @_lib.on_device
    @torch.no_grad()
    def flows(self, enc, pairs, num_flow_updates=None):
        """Flows [len(pairs)][2][H][W] of the frame pairs (i, j) of ``enc`` (flow i -> j)."""
        n_upd = self.num_flow_updates if num_flow_updates is None else int(num_flow_updates)
        pairs = [(int(i), int(j)) for i, j in pairs]
        if any(not 0 <= i < enc.ctx.shape[0] for i, _ in pairs):
            raise _lib.DinotrkError("RAFT: a flow starts from a frame encoded without its context")
        out = torch.empty(len(pairs), 2, enc.H, enc.W, device=self._dev)
        if not pairs:
            return out
        nb = min(self.batch_pairs(enc.H, enc.W), len(pairs))
        ws = self._ws(self._lib.dinotrk_raft_flow_workspace_bytes(enc.H, enc.W, nb))
        st = _lib.stream_ptr()
        for b0 in range(0, len(pairs), nb):
            chunk = pairs[b0:b0 + nb]
            arr = (ctypes.c_int * (2 * len(chunk)))(*[x for p in chunk for x in p])
            _lib.check(self._lib.dinotrk_raft_flow(_lib.ptr(enc.fmap), _lib.ptr(enc.hi), _lib.ptr(enc.lo), _lib.ptr(enc.ctx),
                                                   enc.T, enc.ctx.shape[0], enc.H, enc.W, arr, len(chunk), n_upd,
                                                   ctypes.byref(self._w),
                                                   _lib.ptr(out[b0:b0 + len(chunk)]), _lib.ptr(ws), ws.numel(), st),
                       "raft_flow")
        return out

    def __call__(self, a, b):
        """flow_fn contract: frames a, b [B][3][H][W] in [0, 1] -> flows a -> b [B][2][H][W]."""
        B = a.shape[0]
        enc = self.encode(torch.cat([a.to(self._dev), b.to(self._dev)]), n_context=B)
        return self.flows(enc, [(k, B + k) for k in range(B)])

    def video_flows(self, video01, groups):
        """Encodes the frames of video01 [T][3][H][W] once, then yields the flows [len(g)][2][H][W] of each group g of
        pairs (i, j), lazily."""
        enc = self.encode(video01)
        for g in groups:
            yield self.flows(enc, g)
