#!/usr/bin/env python
"""Phase timeline of the fused MBConv kernels (debug build with -DSYN_FUSED_TRACE, see kernels_fused.cuh).

    nvcc ... -DSYN_FUSED_TRACE -o synergynet_b200/libsynergy_b200_trace.so synergynet_b200/csrc/synergy_b200.cu
    SYN_LIB_PATH=$PWD/synergynet_b200/libsynergy_b200_trace.so python scripts/fused_trace.py 12 2 8

Prints, for CTA 0's second tile of each requested block, clock64 deltas (cycles) per chunk of worker thread 0:
barrier | GEMM1 + EPI1 | barrier | depthwise | barrier + GEMM2."""
import ctypes
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from synergynet_b200 import _lib, synthetic  # noqa: E402
import bench  # noqa: E402


def main():
    blocks = [int(a) for a in sys.argv[1:]] or [2, 12]
    model = bench.build_model('cuda:0')
    x = synthetic.make_inputs(1024, 0).cuda()
    for _ in range(2):
        model.forward_test(x)
    torch.cuda.synchronize()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    n = 18 * 2 * 64 * 8
    buf = (ctypes.c_longlong * n)()
    lib.syn_debug_read_trace(buf, n)
    t = np.frombuffer(buf, dtype=np.int64).reshape(18, 2, 64, 8)
    for b in blocks:
        w = t[b, 0]
        t0 = w[63, 0]
        print(f'== block {b}: tile start 0, chunks done {w[63, 1] - t0}, EPI2 start {w[63, 2] - t0}, EPI2 end {w[63, 4] - t0}')
        q = w[62]
        if q[0]:
            print(f'   prep(next tile): start {q[0] - t0}, staged {q[1] - t0}, all workers {q[2] - t0}, converted {q[3] - t0}, published {q[4] - t0}; first batch: loads issued {q[5] - t0}, first item stored {q[6] - t0}, batch done {q[7] - t0}')
        print('  c | worker: start    bar  G1+EPI1    bar     DW  bar+G2')
        for c in range(62):
            if w[c, 0] == 0:
                break
            wd = [w[c, 1] - w[c, 0], w[c, 3] - w[c, 1], w[c, 4] - w[c, 3], w[c, 5] - w[c, 4], w[c, 6] - w[c, 5]]
            print(f' {c:2d} | {w[c, 0] - t0:13d} {wd[0]:6d} {wd[1]:8d} {wd[2]:6d} {wd[3]:6d} {wd[4]:7d}')


if __name__ == '__main__':
    main()
