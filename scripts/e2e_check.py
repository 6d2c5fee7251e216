#!/usr/bin/env python
"""End-to-end host call, blocking vs two calls in flight, fp32 and uint8 crops: faces/s over 40 steps of 1024 faces."""
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from synergynet_b200 import synthetic  # noqa: E402


def main():
    B, steps = 1024, 40
    model = bench.build_model('cuda:0')
    eng = model._engine(torch.device('cuda', 0))
    outs = [torch.empty((B, 3, 68), dtype=torch.float32).pin_memory() for _ in range(2)]
    res = {}
    for kind, bufs in (('fp32', [synthetic.make_inputs(B, seed=100 + i).pin_memory() for i in range(2)]),
                       ('u8', [synthetic.make_crops_u8(B, seed=100 + i).pin_memory() for i in range(2)])):
        for mode in ('blocking', 'pipelined'):
            for i in range(3):
                eng.forward_landmarks_host(bufs[i % 2], outs[i % 2])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if mode == 'blocking':
                for i in range(steps):
                    eng.forward_landmarks_host(bufs[i % 2], outs[i % 2])
            else:
                prev = None
                for i in range(steps):
                    tk = eng.forward_landmarks_host_submit(bufs[i % 2], outs[i % 2])
                    if prev is not None:
                        eng.host_wait(prev)
                    prev = tk
                eng.host_wait(prev)
            torch.cuda.synchronize()
            res[f'{kind}_{mode}'] = round(B * steps / (time.perf_counter() - t0))
    print(res)


if __name__ == '__main__':
    main()
