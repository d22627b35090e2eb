"""In-tree nvcc build of libdinotrk.so for sm_90a (no JIT cache: the .so travels with the repo)."""
import glob
import os
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG_DIR)
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libdinotrk.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(ROOT, "include", "*.h")) + \
        [os.path.join(ROOT, "tools", "gen_wgmma_ops.py")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile every csrc/*.cu and link libdinotrk.so.  Returns the library path."""
    if not force and not needs_build():
        return LIB_PATH
    objdir = os.path.join(ROOT, "build")
    gendir = os.path.join(objdir, "generated")
    os.makedirs(gendir, exist_ok=True)
    subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gen_wgmma_ops.py"), os.path.join(gendir, "wgmma_ops.cuh")],
                   check=True)
    inc = ["-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-I" + gendir]
    objs, procs = [], []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [_nvcc()] + NVCC_FLAGS + inc + ["-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out.decode()}")
    cmd = [_nvcc(), "-shared", "-o", LIB_PATH] + objs
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout.decode())
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
