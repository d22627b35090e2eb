"""Compare the per-kernel SASS of two builds of libdinotrk.so (CPU only: needs cuobjdump, no GPU).

    python tools/sass_diff.py OLD.so NEW.so

Reports, by mangled name:
  - kernels both builds have whose instruction text differs,
  - kernels only NEW has (a rename when OLD has a kernel with the same instructions),
  - kernels only OLD has (removed, or renamed).
Exits 1 when a common kernel differs or NEW has a kernel with no identical counterpart in OLD, else 0.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_sass_cpu import kernels_sass  # noqa: E402


def main(old_lib, new_lib):
    old = {k: [t for _, t in v] for k, v in kernels_sass(old_lib).items()}
    new = {k: [t for _, t in v] for k, v in kernels_sass(new_lib).items()}
    common = sorted(old.keys() & new.keys())
    changed = [k for k in common if old[k] != new[k]]
    only_old, only_new = sorted(old.keys() - new.keys()), sorted(new.keys() - old.keys())
    same_code = lambda body, pool: [k for k in pool if pool[k] == body]  # noqa: E731
    print(f"{len(old)} kernels in {old_lib}, {len(new)} in {new_lib}")
    print(f"{len(common) - len(changed)} of {len(common)} common kernels have identical SASS")
    for k in changed:
        print(f"  differs: {k} ({len(old[k])} -> {len(new[k])} instructions)")
    new_unmatched = []
    for k in only_new:
        twins = same_code(new[k], {o: old[o] for o in only_old})
        print(f"  only in new: {k}" + (f" (renamed: same SASS as {', '.join(twins)})" if twins else ""))
        if not twins:
            new_unmatched.append(k)
    for k in only_old:
        twins = same_code(old[k], {n: new[n] for n in only_new})
        print(f"  only in old: {k}" + (f" (renamed to {', '.join(twins)})" if twins else " (removed)"))
    return 1 if changed or new_unmatched else 0


if __name__ == "__main__":
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    sys.exit(main(sys.argv[1], sys.argv[2]))
