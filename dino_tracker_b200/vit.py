"""Host mirror of the reference's DINOv2 feature stage (``models/extractor.py::VitExtractor`` +
``utils.py::get_dino_features_video``) over libdinotrk.

The reference builds the backbone with ``torch.hub.load('facebookresearch/dinov2', name)``
(``models/extractor.py:26``), patches its patch-embedding stride to 7 and its position-embedding
interpolation (``:41-85``), runs the video one frame at a time and keeps the output of block ``layer``
before the final norm, cls token dropped (``:137-150``, ``utils.py:54-67``).  Here the weights come from a
DINOv2 state dict (hub key names, so real checkpoints load unchanged), the position embedding is
interpolated once at load time with the reference's formula, and every frame batch is one
``dinotrk_vit_forward`` call that writes token-major features ``[T][P][C]`` directly.  The query / key / value
facets (the reference's qkv hook, ``models/extractor.py:224-266``) and ViT-g/14's SwiGLU feed-forward run on the same
call.  DINO v1's ViT-S/8 and ViT-B/8 (``torch.hub.load('facebookresearch/dino:main', name)`` in the reference) load from
their hub state dict, whose blocks have no LayerScale; their 8-pixel patch comes from the model name, as the reference's
``get_patch_size`` derives it (``models/extractor.py:168-169``).

DINOv2 with registers (hub ``dinov2_vit*14_reg``: the hub keys plus ``register_tokens``) and DINOv3 (``DinoV3Features``:
the state dict of ``transformers``' ``DINOv3ViTModel``) run on the same call.  Their R register tokens sit between cls
and the patches, and DINOv3 replaces the position table by a rotary position embedding (RoPE) on q and k of the patch
tokens.  Its coordinates come from the token grid, so overlapping patches (stride < patch) get the positions the
reference gives DINOv2 by resampling its table onto that grid; at stride = patch they are the hub model's.
"""
import ctypes
import math

import torch
import torch.nn.functional as F

from . import _lib

CONFIGS = {  # name: (depth, dim, heads)
    "dinov2_vits14": (12, 384, 6),
    "dinov2_vitb14": (12, 768, 12),
    "dinov2_vitl14": (24, 1024, 16),
    "dinov2_vitg14": (40, 1536, 24),
    "dino_vits8": (12, 384, 6),
    "dino_vitb8": (12, 768, 12),
    "dinov2_vits14_reg": (12, 384, 6),
    "dinov2_vitb14_reg": (12, 768, 12),
    "dinov2_vitl14_reg": (24, 1024, 16),
    "dinov2_vitg14_reg": (40, 1536, 24),
}
DINOV3_PATCH = 16   # dinov3_vit*16* names: depth, width and heads come from the state dict (DinoV3Features)
_LAYERSCALE = ("ls1.gamma", "ls2.gamma")   # absent from DINO v1 blocks: a null table entry (no LayerScale)
_BLOCK_KEYS = ("norm1.weight", "norm1.bias", "attn.qkv.weight", "attn.qkv.bias", "attn.proj.weight",
               "attn.proj.bias", "ls1.gamma", "norm2.weight", "norm2.bias", "mlp.fc1.weight", "mlp.fc1.bias",
               "mlp.fc2.weight", "mlp.fc2.bias", "ls2.gamma")
# ViT-g/14's SwiGLU feed-forward (hub keys mlp.w12.* / mlp.w3.*) takes slots 9-12 of the weight table
_SWIGLU_KEYS = _BLOCK_KEYS[:9] + ("mlp.w12.weight", "mlp.w12.bias", "mlp.w3.weight", "mlp.w3.bias", "ls2.gamma")
FACETS = {"tokens": 0, "queries": 1, "keys": 2, "values": 3}   # dinotrk_vit_config.facet


def interleave_w12(t):
    """SwiGLU w12 rows (or its bias) from the hub layout [x1 (Hd rows); x2 (Hd rows)] to pairs of hidden units:
    rows 4q .. 4q+3 = x1[2q], x1[2q+1], x2[2q], x2[2q+1].  The CUDA epilogue then finds both halves of an output
    in the same four GEMM columns (dinotrk_vit_weights)."""
    hd = t.shape[0] // 2
    x1, x2 = t[:hd].reshape(hd // 2, 1, 2, *t.shape[1:]), t[hd:].reshape(hd // 2, 1, 2, *t.shape[1:])
    return torch.cat((x1, x2), dim=1).reshape(t.shape).contiguous()


def interpolate_pos_embed(pos_embed, n_h, n_w, square_image=None):
    """models/extractor.py:57-85 (DINOv2 passes (w=H_img, h=W_img)): bicubic, +0.1 trick, align_corners=False,
    recompute_scale_factor=False.  Host-side, once per (model, resolution).  The reference returns the table unchanged
    only when the grid has N tokens AND the frame is square in pixels (``npatch == N and w == h``); ``square_image``
    passes that second condition (None: taken as n_h == n_w, which agrees whenever the frame is square or the grid is
    not N tokens)."""
    N = pos_embed.shape[1] - 1
    dim = pos_embed.shape[-1]
    side = int(math.sqrt(N))
    if n_h * n_w == N and (n_h == n_w if square_image is None else square_image):
        return pos_embed
    cls_pos = pos_embed[:, 0]
    patch_pos = pos_embed[:, 1:].reshape(1, side, side, dim).permute(0, 3, 1, 2)
    w0, h0 = n_h + 0.1, n_w + 0.1
    patch_pos = F.interpolate(patch_pos, scale_factor=(w0 / math.sqrt(N), h0 / math.sqrt(N)), mode="bicubic",
                              align_corners=False, recompute_scale_factor=False)
    assert int(w0) == patch_pos.shape[-2] and int(h0) == patch_pos.shape[-1]
    patch_pos = patch_pos.permute(0, 2, 3, 1).reshape(1, -1, dim)
    return torch.cat((cls_pos[:, None], patch_pos), dim=1)


def patch_size(model_name):
    """models/extractor.py:168-169: 8 for a name containing '8' (DINO v1 ViT-S/8, ViT-B/8), else 14; 16 for DINOv3."""
    if model_name.startswith("dinov3"):
        return DINOV3_PATCH
    return 8 if "8" in model_name else 14


def rope_perm(dim):
    """Row order of q or k that puts head dims (j, j + 32), which RoPE rotates as a pair, in adjacent rows (2j, 2j + 1)
    of every 64-row head: new row i = old row perm[i]."""
    j = torch.arange(32)
    head = torch.stack((j, j + 32), dim=1).reshape(64)
    return (head[None, :] + 64 * torch.arange(dim // 64)[:, None]).reshape(dim)


def rope_table(h, w, theta=100.0, device="cpu"):
    """[h w][32][2] (cos, sin) float32 of DINOv3's rotary embedding on an h x w token grid: coordinates
    2 (i + 0.5) / n - 1 per axis, angles 2 pi coord theta^(-k / 16) for k < 16, y angles first, then x.  Computed in
    float64, rounded once."""
    inv = float(theta) ** (-torch.arange(16, dtype=torch.float64) / 16)
    cy = 2 * (torch.arange(h, dtype=torch.float64) + 0.5) / h - 1
    cx = 2 * (torch.arange(w, dtype=torch.float64) + 0.5) / w - 1
    ay = (2 * math.pi * cy[:, None] * inv)[:, None, :].expand(h, w, 16)
    ax = (2 * math.pi * cx[:, None] * inv)[None, :, :].expand(h, w, 16)
    ang = torch.cat((ay, ax), dim=-1).reshape(h * w, 32)
    return torch.stack((ang.cos(), ang.sin()), dim=-1).to(device, torch.float32).contiguous()


class DinoV2Features(torch.nn.Module):
    """``VitExtractor`` replacement: ``forward(video01)`` -> token-major features [T][P][C] on the GPU.

    ``facet``: 'tokens' (block ``layer``'s output), or 'queries' / 'keys' / 'values' (that block's qkv Linear
    output, the reference's qkv hook, ``models/extractor.py:124-128,224-266``).  A state dict whose blocks carry
    ``mlp.w12.*`` / ``mlp.w3.*`` (ViT-g/14) runs the SwiGLU feed-forward; its hidden width is read from ``w3``.  A state
    dict without ``ls1.gamma`` / ``ls2.gamma`` (DINO v1) runs its blocks without LayerScale.  ``patch`` must match the
    patch embedding's kernel (``from_name`` takes it from the model name).  ``register_tokens`` [1][R][C] in the state
    dict (DINOv2 ``_reg``) puts R register rows after cls.  ``rope_theta`` (DINOv3, see ``DinoV3Features``): no
    position table, RoPE of that base on q and k instead; ``ln_eps``: the LayerNorm eps."""

    def __init__(self, state_dict, heads, layer=None, stride=7, patch=14, device="cuda:0", frames_per_call=2,
                 attention="fused", cta_pairs=True, facet="tokens", rope_theta=None, ln_eps=1e-6):
        super().__init__()
        if facet not in FACETS:
            raise ValueError(f"facet {facet} not supported")
        self.depth = 1 + max(int(k.split(".")[1]) for k in state_dict if k.startswith("blocks."))
        kernel = tuple(state_dict["patch_embed.proj.weight"].shape[-2:])
        if kernel != (patch, patch):
            raise ValueError(f"patch embedding of {kernel} pixels, patch={patch}")
        self.layerscale = "blocks.0.ls1.gamma" in state_dict
        for i in range(self.depth):
            if any((f"blocks.{i}.{k}" in state_dict) != self.layerscale for k in _LAYERSCALE):
                raise ValueError(f"block {i}: LayerScale weights must be present in every block or in none")
        self._dev = _lib.require_cuda(device)
        self._lib = _lib.load()
        sd = {k: v.detach().to(self._dev, torch.float32).contiguous() for k, v in state_dict.items()}
        self.dim = sd["cls_token"].shape[-1]
        self.heads = heads
        self.layer = self.depth - 1 if layer is None else layer
        self.stride, self.patch = stride, patch
        self.frames_per_call = frames_per_call
        assert attention in ("fused", "materialized")
        self.attention = attention
        self.cta_pairs = cta_pairs
        self.facet = facet
        self.swiglu_hidden = self._swiglu_hidden(sd) if "blocks.0.mlp.w12.weight" in sd else 0
        if self.swiglu_hidden:
            for i in range(self.depth):
                for k in ("mlp.w12.weight", "mlp.w12.bias"):
                    sd[f"blocks.{i}.{k}"] = interleave_w12(sd[f"blocks.{i}.{k}"])
        self.n_registers = sd["register_tokens"].shape[1] if "register_tokens" in sd else 0
        self._registers = sd["register_tokens"].reshape(self.n_registers, self.dim).contiguous() if self.n_registers else None
        self.rope_theta, self.ln_eps = rope_theta, float(ln_eps)
        if rope_theta is not None:
            # q and k rows of every head in RoPE pair order (dinotrk_vit_weights); not in the tap block of a facet,
            # whose qkv output is returned as the Linear computes it and whose attention does not run
            perm = torch.cat((rope_perm(self.dim), self.dim + rope_perm(self.dim), torch.arange(2 * self.dim, 3 * self.dim)))
            perm = perm.to(self._dev)
            for i in range(self.depth):
                if not (facet != "tokens" and i == self.layer):
                    for k in ("attn.qkv.weight", "attn.qkv.bias"):
                        sd[f"blocks.{i}.{k}"] = sd[f"blocks.{i}.{k}"][perm].contiguous()
        self._sd = sd
        # fused mode: weight matrices in fp16 (fp16 MMAs); materialized (validation) mode: fp32 / TF32
        self._f16 = attention == "fused"
        wdt = torch.float16 if self._f16 else torch.float32
        mats = ("attn.qkv.weight", "attn.proj.weight", "mlp.fc1.weight", "mlp.fc2.weight", "mlp.w12.weight", "mlp.w3.weight")
        pw = sd["patch_embed.proj.weight"].reshape(self.dim, -1)
        mult = 8 if self._f16 else 4
        if pw.shape[1] % mult:
            pw = F.pad(pw, (0, mult - pw.shape[1] % mult))
        self._patch_w = pw.to(wdt).contiguous()
        keys = _SWIGLU_KEYS if self.swiglu_hidden else _BLOCK_KEYS
        self._blocks = [None if k in _LAYERSCALE and not self.layerscale else
                        sd[f"blocks.{i}.{k}"].to(wdt).contiguous() if k in mats else sd[f"blocks.{i}.{k}"]
                        for i in range(self.depth) for k in keys]
        self._block_ptrs = (ctypes.c_void_p * len(self._blocks))(*[t.data_ptr() if t is not None else None
                                                                    for t in self._blocks])
        self._pos_cache = {}

    def _swiglu_hidden(self, sd):
        """Hd from w3 [D][Hd] (the hub's SwiGLUFFNFused rounds 2/3 of 4 D up to a multiple of 8; not recomputed
        here), and every block's w12 [2 Hd][D] / w3 shapes checked against it."""
        D, hd = self.dim, sd["blocks.0.mlp.w3.weight"].shape[1]
        if hd % 8:
            raise ValueError(f"SwiGLU hidden width {hd} is not a multiple of 8")
        for i in range(self.depth):
            p = f"blocks.{i}.mlp."
            shapes = {k: tuple(sd[p + k].shape) if p + k in sd else None for k in ("w12.weight", "w12.bias", "w3.weight", "w3.bias")}
            want = {"w12.weight": (2 * hd, D), "w12.bias": (2 * hd,), "w3.weight": (D, hd), "w3.bias": (D,)}
            if shapes != want:
                raise ValueError(f"block {i}: SwiGLU weights {shapes}, expected {want}")
        return hd

    @classmethod
    def from_name(cls, model_name, state_dict, **kw):
        """The extractor of a hub model name; a ``dinov3_*`` name gives a ``DinoV3Features`` on a ``transformers``
        state dict (stride 8 unless given)."""
        if model_name.startswith("dinov3"):
            return DinoV3Features(state_dict, patch=patch_size(model_name), **kw)
        depth, dim, heads = CONFIGS[model_name]
        return cls(state_dict, heads=heads, patch=patch_size(model_name), **kw)

    def _pos(self, n_h, n_w, square_image):
        """(cls row, position table [P][D] or None, RoPE table [P][32][2] or None) of an n_h x n_w grid."""
        key = (n_h, n_w, square_image)
        if key not in self._pos_cache:
            if self.rope_theta is not None:
                self._pos_cache[key] = (self._sd["cls_token"].reshape(self.dim).contiguous(), None,
                                        rope_table(n_h, n_w, self.rope_theta, self._dev))
            else:
                pe = interpolate_pos_embed(self._sd["pos_embed"], n_h, n_w, square_image)[0]       # (1 + P) x D
                cls_pos = (self._sd["cls_token"][0, 0] + pe[0]).contiguous()
                self._pos_cache[key] = (cls_pos, pe[1:].contiguous(), None)
        return self._pos_cache[key]

    @torch.no_grad()
    @_lib.on_device
    def forward(self, video01):
        """video01: T x 3 x H x W in [0, 1] (any device).  Returns tpc [T][P][C] (cuda)."""
        lib = self._lib
        T, _, H, W = video01.shape
        geom = _lib.make_geom(H, W, self.patch, self.stride, 35)
        P = geom.h * geom.w
        cfg = _lib.VitConfig(self.depth, self.dim, self.heads, self.layer, self.patch, self.stride,
                             0 if self.attention == "fused" else 1, 1 if self._f16 else 0, 1 if self.cta_pairs else 0,
                             self.swiglu_hidden, FACETS[self.facet])
        cls_pos, pos, rope = self._pos(geom.h, geom.w, H == W)
        wt = _lib.VitWeights()
        wt.patch_w, wt.patch_b = self._patch_w.data_ptr(), self._sd["patch_embed.proj.bias"].data_ptr()
        addr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
        wt.cls_pos, wt.pos = cls_pos.data_ptr(), addr(pos)
        wt.blocks = ctypes.cast(self._block_ptrs, ctypes.POINTER(ctypes.c_void_p))
        wt.registers, wt.n_registers = addr(self._registers), self.n_registers
        wt.rope, wt.ln_eps = addr(rope), self.ln_eps
        out = torch.empty(T, P, self.dim, device=self._dev, dtype=torch.float32)
        B = min(self.frames_per_call, T)
        ws_bytes = lib.dinotrk_vit_workspace_bytes_ext(ctypes.byref(cfg), ctypes.byref(wt), ctypes.byref(geom), B)
        ws = torch.empty(ws_bytes, device=self._dev, dtype=torch.uint8)
        for i in range(0, T, B):
            e = min(i + B, T)
            fr = video01[i:e].to(self._dev, torch.float32).contiguous()
            _lib.check(lib.dinotrk_vit_forward(_lib.ptr(fr), e - i, ctypes.byref(geom), ctypes.byref(cfg), ctypes.byref(wt),
                                               _lib.ptr(out[i:e]), _lib.ptr(ws), ws_bytes, _lib.stream_ptr()), "vit_forward")
        return out

    def features_chw(self, video01):
        """T x C x h x w view (the layout ``dino_embed_video.pt`` stores, utils.py:66)."""
        tpc = self.forward(video01)
        T, P, C = tpc.shape
        geom = _lib.make_geom(video01.shape[-2], video01.shape[-1], self.patch, self.stride, 35)
        return tpc.view(T, geom.h, geom.w, C).permute(0, 3, 1, 2)


def dinov3_to_hub(state_dict):
    """``transformers``' ``DINOv3ViTModel`` state dict -> the DINOv2 hub key layout ``DinoV2Features`` reads: q / k / v
    stacked into ``attn.qkv`` [3C][C] (zero bias where the model has none: k always), ``o_proj`` -> ``attn.proj``,
    ``layer_scale{1,2}.lambda1`` -> ``ls{1,2}.gamma``, ``up_proj`` / ``down_proj`` -> ``mlp.fc1`` / ``mlp.fc2``, or for the
    gated MLP ``[gate_proj; up_proj]`` -> ``mlp.w12`` (silu(gate) up, the SwiGLU path) and ``down_proj`` -> ``mlp.w3``.
    The final norm is not used (the tap is before it)."""
    sd = {k: v.detach() for k, v in state_dict.items()}
    dim = sd["embeddings.cls_token"].shape[-1]
    out = {"cls_token": sd["embeddings.cls_token"].reshape(1, 1, dim),
           "patch_embed.proj.weight": sd["embeddings.patch_embeddings.weight"],
           "patch_embed.proj.bias": sd["embeddings.patch_embeddings.bias"]}
    if sd.get("embeddings.register_tokens") is not None and sd["embeddings.register_tokens"].numel():
        out["register_tokens"] = sd["embeddings.register_tokens"].reshape(1, -1, dim)
    depth = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("model.layer."))
    zeros = lambda n, ref: torch.zeros(n, dtype=ref.dtype, device=ref.device)   # noqa: E731

    def bias(p, n, ref):
        return sd[p + ".bias"] if p + ".bias" in sd else zeros(n, ref)
    for i in range(depth):
        s, d = f"model.layer.{i}.", f"blocks.{i}."
        a = s + "attention."
        ws = [sd[a + f"{x}_proj.weight"] for x in "qkv"]
        out[d + "attn.qkv.weight"] = torch.cat(ws)
        out[d + "attn.qkv.bias"] = torch.cat([bias(a + "q_proj", dim, ws[0]), zeros(dim, ws[0]), bias(a + "v_proj", dim, ws[0])])
        out[d + "attn.proj.weight"] = sd[a + "o_proj.weight"]
        out[d + "attn.proj.bias"] = bias(a + "o_proj", dim, ws[0])
        for n in ("norm1", "norm2"):
            out[d + n + ".weight"], out[d + n + ".bias"] = sd[s + n + ".weight"], sd[s + n + ".bias"]
        out[d + "ls1.gamma"], out[d + "ls2.gamma"] = sd[s + "layer_scale1.lambda1"], sd[s + "layer_scale2.lambda1"]
        m = s + "mlp."
        down = sd[m + "down_proj.weight"]
        hid = down.shape[1]
        if m + "gate_proj.weight" in sd:
            out[d + "mlp.w12.weight"] = torch.cat((sd[m + "gate_proj.weight"], sd[m + "up_proj.weight"]))
            out[d + "mlp.w12.bias"] = torch.cat((bias(m + "gate_proj", hid, down), bias(m + "up_proj", hid, down)))
            out[d + "mlp.w3.weight"], out[d + "mlp.w3.bias"] = down, bias(m + "down_proj", dim, down)
        else:
            out[d + "mlp.fc1.weight"], out[d + "mlp.fc1.bias"] = sd[m + "up_proj.weight"], bias(m + "up_proj", hid, down)
            out[d + "mlp.fc2.weight"], out[d + "mlp.fc2.bias"] = down, bias(m + "down_proj", dim, down)
    return out


class DinoV3Features(DinoV2Features):
    """DINOv3 ViT (``transformers``' ``DINOv3ViTModel`` state dict, which is also what ``from_pretrained`` of the released
    weights gives) on ``DinoV2Features``' call: depth, width, ``heads = C / 64``, the register count and the MLP kind
    (``gate_proj`` present: gated, run as SwiGLU) come from the state dict.  RoPE base ``rope_theta`` (100) on the token
    grid, LayerNorm eps ``ln_eps`` (1e-5).  ``stride`` in [7, patch]: at most 5 tokens across the tracker's 35 px disc; 8
    is the analogue of the reference's 14 / 7, 16 the hub's own grid.  Widths that are not a multiple of 64 (ViT-7B's
    head dim 128) are refused."""

    def __init__(self, state_dict, layer=None, stride=8, patch=DINOV3_PATCH, rope_theta=100.0, ln_eps=1e-5, **kw):
        dim = state_dict["embeddings.cls_token"].shape[-1]
        if dim % 64:
            raise ValueError(f"DINOv3 width {dim} is not a multiple of 64 (head dim 64 only)")
        if not 7 <= stride <= patch:
            raise ValueError(f"stride {stride} outside [7, {patch}]")
        super().__init__(dinov3_to_hub(state_dict), heads=dim // 64, layer=layer, stride=stride, patch=patch,
                         rope_theta=rope_theta, ln_eps=ln_eps, **kw)


@torch.no_grad()
def get_dino_features_video(video, model_name="dinov2_vitb14", facet="tokens", stride=7, layer=None,
                            device="cuda:0", state_dict=None):
    """``utils.py::get_dino_features_video``: T x C x h x w on the CPU like the reference (``utils.py:53,67``), for
    ``facet`` in tokens / queries / keys / values (anything else raises ``ValueError`` as the reference does) and any
    backbone of ``CONFIGS`` (DINOv2 at patch 14, with registers for ``*_reg``, DINO v1 ``dino_vits8`` / ``dino_vitb8`` at patch
    8, ``dinov3_*`` at patch 16 from a ``transformers`` state dict).  ``layer=None``: the
    last block of ``state_dict``.  ``state_dict``: the backbone's weights with hub key names (the reference downloads
    them with torch.hub)."""
    if facet not in FACETS:
        raise ValueError(f"facet {facet} not supported")
    assert state_dict is not None, "pass the backbone's state dict (no network access here)"
    ex = DinoV2Features.from_name(model_name, state_dict, layer=layer, stride=stride, device=device, facet=facet)
    return ex.features_chw(video).cpu()
