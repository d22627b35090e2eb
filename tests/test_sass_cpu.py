"""CPU: no GPU-scope memory fence inside the main loop of any wgmma kernel of libdinotrk.so.

A fence such as MEMBAR.ALL.GPU in a K loop stalls the warpgroup that issues it once per K block.  ptxas emits one for every
release at cluster scope, e.g. an mbarrier arrive written as `.release.cluster` (tc05.cuh, mbar_arrive_cluster); on the
CTA-pair GEMM that fence cost about as much as the K block's MMAs.  The check reads the compiled code.  For every kernel
containing HGMMA, no MEMBAR.*GPU may lie
  - between the first and the last HGMMA in address order, or
  - inside an innermost loop that issues HGMMA: a backward branch whose range holds an HGMMA and no smaller such range
    (ptxas may place the end of the K loop, where a ring slot is released, after the last HGMMA).  Branches after the
    last EXIT do not count: they return from the out-of-line retry paths of barrier waits, and are not loops.
Fences in a prologue (barrier initialisation) or at the exit (the final cluster barrier) are outside both and allowed.
Needs nvcc and cuobjdump, no GPU.
"""
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
HGMMA = re.compile(r"\bHGMMA\b")
GPU_FENCE = re.compile(r"\bMEMBAR\b\S*\.GPU\b")
BRANCH = re.compile(r"\bBRA\b.*?(0x[0-9a-f]+)\s*$")


def _cuobjdump():
    from dino_tracker_b200 import build as b
    nvcc = b._nvcc()
    cand = os.path.join(os.path.dirname(nvcc), "cuobjdump") if os.path.isabs(nvcc) else None
    return cand if cand and os.path.exists(cand) else shutil.which("cuobjdump")


def kernels_sass(lib):
    """{mangled kernel name: [(address, instruction text)]} of the sm_90a code in `lib`."""
    out = subprocess.run([_cuobjdump(), "-sass", lib], check=True, stdout=subprocess.PIPE, text=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        s = line.strip()
        if s.startswith("Function : "):
            cur = funcs.setdefault(s[len("Function : "):], [])
        elif cur is not None:
            m = INSN.match(line)
            if m:
                cur.append((int(m.group(1), 16), m.group(2)))
    return funcs


def gpu_fences_in_mma_loop(insns):
    """The MEMBAR.*GPU instructions (address, text) of a kernel that lie in its wgmma main loop (see the module doc)."""
    hg = [a for a, t in insns if HGMMA.search(t)]
    if not hg:
        return []
    ranges = [(min(hg), max(hg))]
    body_end = max((a for a, t in insns if re.search(r"\bEXIT\b", t)), default=insns[-1][0])
    loops = []
    for a, t in insns:
        m = BRANCH.search(t)
        if m and a < body_end and int(m.group(1), 16) <= a and any(int(m.group(1), 16) <= h <= a for h in hg):
            loops.append((int(m.group(1), 16), a))
    ranges += [(lo, hi) for lo, hi in loops
               if not any((l2, h2) != (lo, hi) and lo <= l2 and h2 <= hi for l2, h2 in loops)]
    return [(a, t) for a, t in insns if GPU_FENCE.search(t) and any(lo <= a <= hi for lo, hi in ranges)]


def test_no_gpu_fence_inside_wgmma_loops():
    from dino_tracker_b200 import build as b
    assert _cuobjdump(), "cuobjdump not found next to nvcc or on PATH"
    funcs = kernels_sass(b.build())
    with_hgmma = [k for k, v in funcs.items() if any(HGMMA.search(t) for _, t in v)]
    assert with_hgmma, "no HGMMA kernel found in libdinotrk.so"
    bad = {k: gpu_fences_in_mma_loop(funcs[k]) for k in with_hgmma}
    bad = {k: v for k, v in bad.items() if v}
    msg = "\n".join(f"  {k}: " + ", ".join(f"{t} @0x{a:x}" for a, t in v) for k, v in bad.items())
    assert not bad, "GPU-scope fence in the wgmma main loop of:\n" + msg
