"""ViT-L/14 (stride 7, 854x476, tap at block 15) feature-extraction stage on its own: device time per frame and the
per-class kernel times.  GPU only."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--C", type=int, default=1024)
    a = ap.parse_args()
    from dino_tracker_b200 import _lib
    _lib.load()
    r = bench.stage_timings(a, "cuda:0", _lib, bench.measured_peaks(), vit_only=True)
    print(json.dumps(r["vit"]))


if __name__ == "__main__":
    main()
