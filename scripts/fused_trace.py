#!/usr/bin/env python
"""Phase timeline of the fused MBConv kernels (debug build with -DSYN_FUSED_TRACE, see kernels_fused.cuh).

    nvcc ... -DSYN_FUSED_TRACE -o synergynet_b200/libsynergy_b200_trace.so synergynet_b200/csrc/synergy_b200.cu
    SYN_LIB_PATH=$PWD/synergynet_b200/libsynergy_b200_trace.so python scripts/fused_trace.py 12 2 8

Prints, for CTA 0's second tile of each requested block, clock64 deltas (cycles) per chunk of worker thread 0:
barrier | GEMM1 + EPI1 | barrier | depthwise | barrier + GEMM2.  Block 1 (stem_block1_kernel, kernels_stem.cuh) is
shown per strip pipeline instead: CTA 0's second strip of each pipeline, phases prep (of the next strip) | GEMM1 + EPI1 |
depthwise | GEMM2 | EPI2, on the SM's common clock so that the two pipelines' phases can be laid side by side."""
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
        if b == 1 and t[1, 1, 63, 0]:
            stem(t[1])
            continue
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



def stem(t):
    """Rows 63 (the strip) and 62 (the prep of the pipeline's next strip) of both pipelines, from pipeline 0's start."""
    t0 = t[0, 63, 0]
    print('== block 1 (stem kernel): cycles from pipeline 0\'s strip start')
    print(' pl | start  window  G1+EPI1    bar     DW  bar+G2 | prep: stage    bar  im2col | EPI2    end')
    for pl in range(2):
        w, q = t[pl, 63], t[pl, 62]
        d = [w[1] - w[0], w[2] - w[1], w[3] - w[2], w[4] - w[3], w[5] - w[4]]
        pr = [q[1] - q[0], q[2] - q[1], q[3] - q[2]] if q[0] else [0, 0, 0]
        print(f'  {pl} | {w[0] - t0:5d} {d[0]:7d} {d[1]:8d} {d[2]:6d} {d[3]:6d} {d[4]:7d} | {pr[0]:11d} {pr[1]:6d} {pr[2]:7d} '
              f'| {w[7] - w[6]:5d} {w[7] - t0:6d}')


if __name__ == '__main__':
    main()
