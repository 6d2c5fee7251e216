#!/usr/bin/env python
"""Timeline of dense_recon_fm_kernel's CTA 0 (SYN_DENSE_TRACE=<file> makes the library dump clock64 stamps), cycles:
loader per item: [plane 0 / 1 / 2 requested (its ring slot was free)]; team 0 (thread 0) per item:
[wait alpha + meta | MMAs of the three planes done | staged + stored]."""
import sys

rows = [l.split() for l in open(sys.argv[1])]
ep = {(r[0], int(r[1])): [int(x) for x in r[2:]] for r in rows}
t0 = min(v[0] for v in ep.values() if v[0] > 0)
print(' item | loader: plane0  plane1  plane2 | team 0: start  w.meta   mma  stored')
for i in range(0, 64):
    ld = ep.get(('loader', i)); e = ep.get(('team0', i))
    if not e or e[0] == 0:
        break
    pl = [f'{v - t0:7d}' if ld and v else '      -' for v in (ld[:3] if ld else [0, 0, 0])]
    print(f' {i:4d} | {" ".join(pl)} | {e[0] - t0:13d} {e[1] - e[0]:7d} {e[2] - e[1]:5d} {e[4] - e[2]:7d}')
