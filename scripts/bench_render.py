"""Sim3DR / FaceBoxes post-processing measurement alone (the `render` / `detect` objects of bench.py's line):
    python scripts/bench_render.py [--no-cpu]  > render_bench.json"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

if __name__ == '__main__':
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    out = bench.render_detect_measurement(dev, bench.load_peaks(), cpu_too='--no-cpu' not in sys.argv)
    print(json.dumps(out))
