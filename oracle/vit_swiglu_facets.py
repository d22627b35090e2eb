"""Oracle restatement of the DINOv2 feature stage beyond ``oracle/vit.py``: ViT-g/14's SwiGLU feed-forward and the
query / key / value facets (SURVEY.md 8a row a1).

Test infrastructure (see ``oracle/__init__.py``).  ``oracle/vit.py`` stays the oracle of the GELU backbones and of the
'tokens' facet; this module reuses its stem pieces and adds:

* the SwiGLU MLP of facebookresearch/dinov2's ``SwiGLUFFNFused`` (ViT-g/14's ``ffn_layer``): ``w12`` [2 Hd][D], chunk
  into (x1, x2), ``silu(x1) * x2``, then ``w3`` [D][Hd], with Hd = ``(int(4 D * 2 / 3) + 7) // 8 * 8`` (4096 for
  D = 1536), in the hub's (non-interleaved) layout.  Cross-checked against ``transformers``' Dinov2Layer with
  ``use_swiglu_ffn=True`` (tests/test_vit_swiglu_facets_oracle_cpu.py);
* the facets: the reference hooks block ``layer``'s ``attn.qkv`` Linear and reshapes its output to (B, N, 3, C), so
  queries / keys / values are rows [0, C), [C, 2C), [2C, 3C) of that Linear's output, unscaled
  (models/extractor.py:124-128,224-266; utils.py:57-64).  Pinned by ``tests/golden/vit_facets_small.npz`` and
  ``vit_g_small.npz`` from the live reference (``oracle/make_golden_vit_models.py``).
"""
import torch
import torch.nn.functional as F

from . import vit as ovit

CONFIGS = {**ovit.CONFIGS, "dinov2_vitg14": (40, 1536, 24)}   # name: (depth, dim, heads)
FACETS = ("tokens", "queries", "keys", "values")


def swiglu_hidden(dim):
    """Hidden width of the hub's SwiGLUFFNFused at mlp_ratio 4."""
    return (int(4 * dim * 2 / 3) + 7) // 8 * 8


def random_state_dict(depth, dim, gen, n_pos=37, patch=14, ls_init=1.0, std=0.02, swiglu=False):
    """``oracle.vit.random_state_dict``, or with ``swiglu`` the same draws with ``mlp.w12.*`` / ``mlp.w3.*`` in place
    of ``mlp.fc1.*`` / ``mlp.fc2.*``."""
    if not swiglu:
        return ovit.random_state_dict(depth, dim, gen, n_pos, patch, ls_init, std)
    hd = swiglu_hidden(dim)

    def tn(*shape):
        return torch.randn(*shape, generator=gen) * std
    sd = ovit.random_state_dict(0, dim, gen, n_pos, patch, ls_init, std)
    for i in range(depth):
        p = f"blocks.{i}."
        sd[p + "norm1.weight"] = 1 + tn(dim); sd[p + "norm1.bias"] = tn(dim)
        sd[p + "attn.qkv.weight"] = tn(3 * dim, dim) * 2; sd[p + "attn.qkv.bias"] = tn(3 * dim)
        sd[p + "attn.proj.weight"] = tn(dim, dim); sd[p + "attn.proj.bias"] = tn(dim)
        sd[p + "ls1.gamma"] = torch.full((dim,), ls_init) + tn(dim)
        sd[p + "norm2.weight"] = 1 + tn(dim); sd[p + "norm2.bias"] = tn(dim)
        sd[p + "mlp.w12.weight"] = tn(2 * hd, dim); sd[p + "mlp.w12.bias"] = tn(2 * hd)
        sd[p + "mlp.w3.weight"] = tn(dim, hd); sd[p + "mlp.w3.bias"] = tn(dim)
        sd[p + "ls2.gamma"] = torch.full((dim,), ls_init) + tn(dim)
    return sd


def qkv(x, sd, i):
    """Block i's ``attn.qkv`` Linear on its LayerNorm-1 output: B x N x 3D (what the reference's qkv hook records)."""
    p = f"blocks.{i}."
    y = F.layer_norm(x, (x.shape[-1],), sd[p + "norm1.weight"], sd[p + "norm1.bias"], eps=1e-6)
    return F.linear(y, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"])


def block_forward(x, sd, i, heads):
    """One DINOv2 block: ``oracle.vit.block_forward`` for the GELU MLP, else attention as there + the SwiGLU MLP."""
    p = f"blocks.{i}."
    if p + "mlp.w12.weight" not in sd:
        return ovit.block_forward(x, sd, i, heads)
    B, N, D = x.shape
    hd = D // heads
    t = qkv(x, sd, i).reshape(B, N, 3, heads, hd).permute(2, 0, 3, 1, 4)
    q, k, v = t[0] * hd ** -0.5, t[1], t[2]
    y = (torch.softmax(q @ k.transpose(-2, -1), dim=-1) @ v).transpose(1, 2).reshape(B, N, D)
    x = x + F.linear(y, sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"]) * sd[p + "ls1.gamma"]
    y = F.layer_norm(x, (D,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], eps=1e-6)
    x1, x2 = F.linear(y, sd[p + "mlp.w12.weight"], sd[p + "mlp.w12.bias"]).chunk(2, dim=-1)
    y = F.linear(F.silu(x1) * x2, sd[p + "mlp.w3.weight"], sd[p + "mlp.w3.bias"])
    return x + y * sd[p + "ls2.gamma"]


def vit_tokens(frames01, sd, heads, layer, stride=7, patch=14, facet="tokens"):
    """frames01: B x 3 x H x W in [0, 1].  'tokens': block ``layer``'s output B x (1 + h w) x D; a facet: that block's
    query / key / value rows of its qkv Linear output, B x (1 + h w) x D."""
    if facet not in FACETS:
        raise ValueError(f"facet {facet} not supported")
    mean = torch.tensor(ovit.IMAGENET_MEAN, device=frames01.device)[None, :, None, None]
    std = torch.tensor(ovit.IMAGENET_STD, device=frames01.device)[None, :, None, None]
    x = F.conv2d((frames01 - mean) / std, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=stride)
    B, D, n_h, n_w = x.shape
    x = torch.cat((sd["cls_token"].expand(B, -1, -1), x.flatten(2).transpose(1, 2)), dim=1)
    x = x + ovit.interpolate_pos_embed(sd["pos_embed"], n_h, n_w)
    for i in range(layer):
        x = block_forward(x, sd, i, heads)
    if facet == "tokens":
        return block_forward(x, sd, layer, heads)
    f = FACETS.index(facet) - 1
    return qkv(x, sd, layer)[..., f * D:(f + 1) * D]


def dino_features_video(video01, sd, heads, layer, stride=7, patch=14, facet="tokens"):
    """utils.py:32-72: per-frame loop, cls dropped, -> T x C x h x w."""
    T, _, H, W = video01.shape
    ph, pw = 1 + (H - patch) // stride, 1 + (W - patch) // stride
    out = []
    for i in range(T):
        tok = vit_tokens(video01[i:i + 1], sd, heads, layer, stride, patch, facet)
        out.append(tok[0, 1:].reshape(ph, pw, -1).permute(2, 0, 1))
    return torch.stack(out)
