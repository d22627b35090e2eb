"""Write tests/golden/vit_dinov3_small.npz: ``transformers``' DINOv3ViTModel run in float64 on seeded weights (the
state dicts of ``oracle.vit_dinov3.random_state_dict``) and seeded videos, block ``layer``'s output with cls and registers
dropped, T x C x h x w at stride = patch = 16.  The GPU tests compare the CUDA feature stage with it, so they never need
``transformers``.

    python -m oracle.make_golden_vit_dinov3
"""
import os

import numpy as np
import torch

from . import synth
from . import vit_dinov3 as ov3

CASES = [
    dict(name="gelu_r4", depth=2, dim=128, registers=4, gated=False, hidden=512, seed=11, frames=2, H=64, W=96, layer=1),
    dict(name="gated_r0", depth=2, dim=128, registers=0, gated=True, hidden=344, seed=12, frames=2, H=70, W=100, layer=1),
]
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "vit_dinov3_small.npz")


def case_state_dict(case):
    return ov3.random_state_dict(case["depth"], case["dim"], torch.Generator().manual_seed(case["seed"]),
                                 registers=case["registers"], gated=case["gated"], hidden=case["hidden"], std=0.05)


def case_video(case):
    return synth.random_video(case["frames"], case["H"], case["W"], seed=case["seed"] + 100)


def run_transformers(case):
    import transformers
    cfg = transformers.DINOv3ViTConfig(hidden_size=case["dim"], num_hidden_layers=case["depth"],
                                       num_attention_heads=case["dim"] // 64, intermediate_size=case["hidden"],
                                       num_register_tokens=case["registers"], patch_size=16, use_gated_mlp=case["gated"],
                                       hidden_act="silu" if case["gated"] else "gelu", layer_norm_eps=1e-5,
                                       rope_theta=100.0, key_bias=False)
    m = transformers.DINOv3ViTModel(cfg).double().eval()
    m.load_state_dict({k: v.double() for k, v in case_state_dict(case).items()}, strict=False)
    video = case_video(case).double()
    with torch.no_grad():
        hs = m(pixel_values=ov3.normalize(video), output_hidden_states=True).hidden_states[case["layer"] + 1]
    h, w = case["H"] // 16, case["W"] // 16
    return hs[:, 1 + case["registers"]:].reshape(case["frames"], h, w, -1).permute(0, 3, 1, 2).contiguous()


def main():
    np.savez_compressed(OUT, **{c["name"]: run_transformers(c).numpy() for c in CASES})
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
