"""Parameter containers with the reference's state-dict keys + host-side weight preparation.

``DeltaDINO`` mirrors ``models/networks/delta_dino.py`` (keys ``layers.{0,4,8,12}.{weight,bias}``,
``layers.{1,5,9,13}.*`` BatchNorm, ``layers.{3,7,11}.filt``) and ``TrackerHead`` mirrors
``models/networks/tracker_head.py`` (keys ``cnn_refiner.{0,2}.{weight,bias}``), so the reference's
checkpoints load bit-for-bit.  Without autograd neither module runs torch arithmetic: they fold / normalise their
weights once per parameter version and hand them to the CUDA kernels.  With autograd (the training step,
``dino_tracker.py:405-429``) the refiner's weight normalisation is a torch graph; delta-DINO is one autograd node with
CUDA forward and backward (``train.DeltaTrainFunction``) when its widths are multiples of 8, and a torch graph
(``forward_graph``: cuDNN convolutions, BatchNorm in the module's mode) otherwise.
"""
import ctypes
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from . import train as _train


class NormalizedConv2d(nn.Module):
    """Parameter holder of ``models/networks/conv_norm.py`` (weights are divided by their spatial sum)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels, kernel_size, kernel_size))
        self.bias = nn.Parameter(torch.empty(out_channels))
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        fan_in = in_channels * kernel_size * kernel_size
        nn.init.uniform_(self.bias, -1 / math.sqrt(fan_in), 1 / math.sqrt(fan_in))

    def normalized_weight_graph(self):
        """The same normalisation as a torch graph on the parameter's device (training: the gradient of the
        normalised weights, produced by ``dinotrk_track_backward``, flows back to ``weight`` through it)."""
        s = self.weight.sum(dim=[2, 3], keepdim=True)
        s = torch.where(s.abs() < 1e-8, torch.sign(s) * 1e-8, s)
        return self.weight / s

    def normalized_weight(self):
        """conv_norm.py:34-46: w / sum_{3x3} w, |sum| < 1e-8 -> sign(sum) * 1e-8."""
        w = self.weight.detach().to("cpu", torch.float32)
        s = w.sum(dim=[2, 3])[:, :, None, None].clone()
        unstable = s.abs() < 1e-8
        if unstable.any():
            s[unstable] = torch.sign(s[unstable]) * 1e-8
        return w / s


class TrackerHead(nn.Module):
    def __init__(self, use_cnn_refiner=True, in_channels=1, hidden_channels=16, out_channels=1, kernel_size=3,
                 stride=1, patch_size=14, step_h=14, step_w=14, argmax_radius=35, video_h=480, video_w=640):
        super().__init__()
        assert use_cnn_refiner and in_channels == 1 and hidden_channels == 16 and out_channels == 1 and kernel_size == 3
        pad = kernel_size // 2
        self.cnn_refiner = nn.Sequential(NormalizedConv2d(in_channels, hidden_channels, kernel_size, stride, pad),
                                         nn.ReLU(inplace=True),
                                         NormalizedConv2d(hidden_channels, out_channels, kernel_size, stride, pad))
        self.argmax_radius = argmax_radius
        self.patch_size, self.step_h, self.step_w = patch_size, step_h, step_w
        self.video_h, self.video_w = video_h, video_w

    def packed_weights(self) -> _lib.HeadWeights:
        hw = _lib.HeadWeights()
        w1 = self.cnn_refiner[0].normalized_weight().reshape(16, 9)
        w2 = self.cnn_refiner[2].normalized_weight().reshape(16, 9)
        b1 = self.cnn_refiner[0].bias.detach().to("cpu", torch.float32)
        b2 = self.cnn_refiner[2].bias.detach().to("cpu", torch.float32)
        for o in range(16):
            for k in range(9):
                hw.w1[o][k] = float(w1[o, k])
                hw.w2[o][k] = float(w2[o, k])
            hw.b1[o] = float(b1[o])
        hw.b2 = float(b2[0])
        return hw


class _BlurPoolParams(nn.Module):
    """Holds the ``filt`` buffer of antialiased_cnns.BlurPool (C x 1 x 4 x 4) for checkpoint parity."""

    def __init__(self, channels):
        super().__init__()
        a = torch.tensor([1.0, 3.0, 3.0, 1.0])
        f = a[:, None] * a[None, :]
        self.register_buffer("filt", (f / f.sum())[None, None].repeat(channels, 1, 1, 1))

    def forward(self, x):
        """Autograd (training) path only: reflect pad (1, 2, 1, 2), depthwise 4 x 4 binomial filter, stride 2."""
        return F.conv2d(F.pad(x, (1, 2, 1, 2), mode="reflect"), self.filt, stride=2, groups=x.shape[1])


class DeltaDINO(nn.Module):
    def __init__(self, channels=(3, 64, 128, 256, 1024), dilations=(1, 1, 1, 2), kernel_size=5, down_stride=2,
                 padding_mode="reflect", downsample_layers=(True, True, True, False), vit_stride=7,
                 conv_precision=None):
        super().__init__()
        channels = list(channels)
        assert len(channels) == 5 and kernel_size == 5 and tuple(dilations) == (1, 1, 1, 2)
        self.channels = channels
        self.vit_stride = vit_stride
        self.down_stride = down_stride
        layers = []
        for i in range(4):
            last = i == 3
            conv = nn.Conv2d(channels[i], channels[i + 1], 5, stride=1, dilation=dilations[i],
                             padding=(5 + 4 * (dilations[i] - 1)) // 2, padding_mode=padding_mode)
            if last:  # zero init, models/networks/delta_dino.py:32-34
                nn.init.zeros_(conv.weight); nn.init.zeros_(conv.bias)
            layers.append(conv)
            bn = nn.BatchNorm2d(channels[i + 1])
            if last:
                bn.weight.data.fill_(0.05)
            layers.append(bn)
            if not last:
                layers.append(nn.ReLU())
                layers.append(_BlurPoolParams(channels[i + 1]))
        self.layers = nn.ModuleList(layers)
        self._folded = (None, None)
        # "fp16x3": convolutions as im2col + wgmma split-precision GEMMs (needs channel counts % 8 == 0);
        # "fp32": exact-fp32 implicit GEMM on the CUDA cores
        ok8 = all(c % 8 == 0 for c in channels[1:])
        self.conv_precision = conv_precision or ("fp16x3" if ok8 else "fp32")
        assert self.conv_precision in ("fp16x3", "fp32") and (ok8 or self.conv_precision == "fp32")

    def get_total_stride(self):
        return self.down_stride ** 3

    def _fold(self):
        """BatchNorm(eval) folded into K-major conv weights [C_out][5][5][C_in_pad] (+ bias)."""
        key = tuple((p.data_ptr(), p._version) for p in list(self.parameters()) + list(self.buffers()))
        if self._folded[0] == key:
            return self._folded[1]
        ws, bs = [], []
        for li, (ci, bi) in enumerate(zip((0, 4, 8, 12), (1, 5, 9, 13))):
            conv, bn = self.layers[ci], self.layers[bi]
            scale = bn.weight.detach() / torch.sqrt(bn.running_var + bn.eps)
            w = conv.weight.detach() * scale[:, None, None, None]
            b = (conv.bias.detach() - bn.running_mean) * scale + bn.bias.detach()
            w = w.permute(0, 2, 3, 1)  # O, ky, kx, I
            if w.shape[-1] % 4:
                w = torch.nn.functional.pad(w, (0, 4 - w.shape[-1] % 4))
            ws.append(w.contiguous().float())
            bs.append(b.contiguous().float())
        # fp16 hi / lo split of the K-major weights, K padded to a multiple of 8 (tensor-core path)
        his, los = [], []
        if self.conv_precision == "fp16x3":
            lib = _lib.load()
            for w in ws:
                w2 = w.reshape(w.shape[0], -1)
                if w2.shape[1] % 8:
                    w2 = torch.nn.functional.pad(w2, (0, 8 - w2.shape[1] % 8))
                w2 = w2.contiguous()
                hi = torch.empty(w2.shape, device=w2.device, dtype=torch.float16)
                lo = torch.empty(w2.shape, device=w2.device, dtype=torch.float16)
                _lib.check(lib.dinotrk_split_fp16(_lib.ptr(w2), _lib.ptr(hi), _lib.ptr(lo), w2.numel(), _lib.stream_ptr()))
                his.append(hi); los.append(lo)
        self._folded = (key, (ws, bs, his, los))
        return ws, bs, his, los

    @staticmethod
    def align_tables(cnn_hw, vit_hw, device, vit_patch_size=14, vit_stride=7, cnn_stride=8):
        """Per-axis source coordinates of models/utils.py:31-43 + grid_sample's un-normalisation
        (align_corners=True, border), in the reference's fp32 arithmetic."""
        out = []
        for n_c, n_v in ((cnn_hw[1], vit_hw[1]), (cnn_hw[0], vit_hw[0])):
            c_br = (n_c - 1) * cnn_stride
            v = torch.arange(n_v, dtype=torch.float32) * vit_stride + vit_patch_size / 2.
            g = -1. - (1. / c_br) + (2. * v / c_br)
            src = ((g + 1) / 2) * (n_c - 1)
            out.append(src.clamp(0, n_c - 1).to(device).contiguous())
        return out  # ixs [w], iys [h]

    @torch.no_grad()
    def refine_tpc(self, frames, dino_tpc, geom, batch=8, out=None, peer_ptrs=None, first_frame=0):
        """frames B x 3 x H x W, dino_tpc [B][P][C] -> (refined_tpc, norms) via dinotrk_delta_refine,
        in batches of 8 frames like models/tracker.py:118-123.  ``out``: write the refined rows there ([B][P][C]
        view, e.g. this rank's slice of a full feature video); ``peer_ptrs`` (+ ``first_frame``): also store every
        row into the peers' full buffers from inside the producing kernel (fused all-gather over NVLink)."""
        lib = _lib.load()
        dev = dino_tpc.device
        ws, bs, his, los = self._fold()
        tensor = self.conv_precision == "fp16x3"
        B, _, H, W = frames.shape
        C = self.channels[-1]
        assert dino_tpc.shape[-1] == C, f"DeltaDINO emits {C} channels, features have {dino_tpc.shape[-1]}"
        ch, cw = H, W
        for _ in range(3):
            ch, cw = (ch - 1) // 2 + 1, (cw - 1) // 2 + 1
        ixs, iys = self.align_tables((ch, cw), (geom.h, geom.w), dev, vit_stride=self.vit_stride)
        chan = (ctypes.c_int * 5)(*self.channels)
        wp = (ctypes.c_void_p * 4)(*[w.data_ptr() for w in ws])
        bp = (ctypes.c_void_p * 4)(*[b.data_ptr() for b in bs])
        if tensor:
            whp = (ctypes.c_void_p * 4)(*[w.data_ptr() for w in his])
            wlp = (ctypes.c_void_p * 4)(*[w.data_ptr() for w in los])
        refined = torch.empty_like(dino_tpc) if out is None else out
        assert refined.is_contiguous() and refined.shape == dino_tpc.shape
        norms = torch.empty(dino_tpc.shape[:2], device=dev, dtype=torch.float32)
        peers = None
        if peer_ptrs:
            peers = (ctypes.c_void_p * len(peer_ptrs))(*peer_ptrs)
        nb = min(batch, B)
        ws_bytes = lib.dinotrk_delta_workspace_bytes(nb, H, W, chan)
        work = torch.empty(ws_bytes, device=dev, dtype=torch.uint8)
        for i in range(0, B, batch):
            e = min(i + batch, B)
            fr = frames[i:e].contiguous()
            if tensor:
                _lib.check(lib.dinotrk_delta_refine_tc(
                    _lib.ptr(fr), e - i, H, W, chan, whp, wlp, bp, _lib.ptr(dino_tpc[i:e]), _lib.ptr(ixs), _lib.ptr(iys),
                    geom.h, geom.w, _lib.ptr(refined[i:e]), _lib.ptr(norms[i:e]), _lib.ptr(work), ws_bytes,
                    peers, len(peer_ptrs) if peer_ptrs else 0, first_frame + i, _lib.stream_ptr()), "delta_refine_tc")
            elif peers is None:
                _lib.check(lib.dinotrk_delta_refine(
                    _lib.ptr(fr), e - i, H, W, chan, wp, bp, _lib.ptr(dino_tpc[i:e]), _lib.ptr(ixs), _lib.ptr(iys),
                    geom.h, geom.w, _lib.ptr(refined[i:e]), _lib.ptr(norms[i:e]), _lib.ptr(work), ws_bytes,
                    _lib.stream_ptr()), "delta_refine")
            else:
                _lib.check(lib.dinotrk_delta_refine_allgather(
                    _lib.ptr(fr), e - i, H, W, chan, wp, bp, _lib.ptr(dino_tpc[i:e]), _lib.ptr(ixs), _lib.ptr(iys),
                    geom.h, geom.w, _lib.ptr(refined[i:e]), _lib.ptr(norms[i:e]), _lib.ptr(work), ws_bytes,
                    peers, len(peer_ptrs), first_frame + i, _lib.stream_ptr()), "delta_refine_allgather")
        return refined, norms

    def wants_graph(self):
        return torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())

    def forward_graph(self, x, vit_hw, vit_patch_size=14):
        """Training path of models/networks/delta_dino.py:53-61 as a torch graph: the layer stack (BatchNorm in the
        module's current mode) and the bilinear alignment of models/utils.py:7-45 (grid without gradient)."""
        for layer in self.layers:
            x = layer(x)
        n_h, n_w = x.shape[-2:]
        cnn_stride = self.get_total_stride()
        axes = []
        for n_c, n_v in ((n_w, vit_hw[1]), (n_h, vit_hw[0])):
            c_br = (n_c - 1) * cnn_stride
            v = torch.arange(n_v, dtype=x.dtype, device=x.device) * self.vit_stride + vit_patch_size / 2.
            axes.append(-1. - (1. / c_br) + (2. * v / c_br))
        gx, gy = torch.meshgrid(axes[0], axes[1], indexing="xy")
        grid = torch.stack([gx, gy], dim=-1)[None].expand(x.shape[0], -1, -1, -1)
        return F.grid_sample(x, grid=grid, mode="bilinear", padding_mode="border", align_corners=True)

    def forward(self, x, vit_features):
        """models/networks/delta_dino.py:53-61: returns the aligned residual B x C x h x w."""
        if self.wants_graph():
            if self.conv_precision == "fp16x3":      # the widths the tensor-core convolutions take (as inference)
                return _train.delta_train(self, x.float(), vit_features.shape[-2:])
            return self.forward_graph(x.float(), vit_features.shape[-2:])
        B, C, h, w = vit_features.shape
        geom = _lib.make_geom(x.shape[-2], x.shape[-1], 14, self.vit_stride, 35)
        geom.h, geom.w = h, w   # the backbone's grid: patch-14 alignment, but 16-pixel patches have fewer columns
        zeros = torch.zeros(B, h * w, C, device=vit_features.device, dtype=torch.float32)
        res, _ = self.refine_tpc(x.float().contiguous(), zeros, geom)
        return res.view(B, h, w, C).permute(0, 3, 1, 2)
