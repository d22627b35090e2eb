"""CPU: the int8 coarse-pass GEMM (tc_gemm_pair_kernel<S8, ...>) issues integer wgmma (IGMMA) and has no GPU-scope memory
fence in its main loop -- the check test_sass_cpu.py makes for the HGMMA kernels, on the IGMMA one.  Needs nvcc and
cuobjdump, no GPU."""
import importlib.util
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
IGMMA = re.compile(r"\bIGMMA\b")
S8_KERNEL = "tc_gemm_pair_kernelILNS_6TcModeE5E"   # mangled prefix of tc_gemm_pair_kernel<TcMode::S8, ...>


def _sass_module():
    spec = importlib.util.spec_from_file_location("sass_check", os.path.join(HERE, "test_sass_cpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_int8_coarse_gemm_uses_igmma_without_gpu_fence_in_loop():
    from dino_tracker_b200 import build as b
    sass = _sass_module()
    assert sass._cuobjdump(), "cuobjdump not found next to nvcc or on PATH"
    funcs = sass.kernels_sass(b.build())
    s8 = {k: v for k, v in funcs.items() if S8_KERNEL in k}
    assert s8, "no int8 coarse GEMM kernel in libdinotrk.so"
    for name, insns in s8.items():
        assert any(IGMMA.search(t) for _, t in insns), f"{name}: no IGMMA"
        assert not any(re.search(r"\bHGMMA\b", t) for _, t in insns), f"{name}: floating-point wgmma in the int8 kernel"
        # the loop analysis of test_sass_cpu.py keys on HGMMA: present the integer MMAs to it under that name
        as_h = [(a, IGMMA.sub("HGMMA", t)) for a, t in insns]
        bad = sass.gpu_fences_in_mma_loop(as_h)
        assert not bad, f"{name}: GPU-scope fence in the wgmma main loop: {bad}"
