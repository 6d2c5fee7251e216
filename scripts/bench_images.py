"""Image-list measurement: the ``*_images`` path on images of mixed sizes against a loop of the one-image calls on the
same images, in one command.
    python scripts/bench_images.py [--counts 1,4,16,64] > images_bench.json

Images: seeded synthetic.make_scene_u8 scenes with sizes drawn (seed 5) from 450x450, 480x640, 720x1080, 1080x1920 and
300x400 -- photo-collection sizes, 1080x1920 above the detector's 720x1080 limit, so it is shrunk on the device.
Detector weights: synthetic.make_faceboxes_state_dict(0); backbone: bench.py's seeded mobilenet_v2.  For every image
count N, every shape warmed up first and the two paths alternating round by round (bench_frames.py's timers):
  network_ms_per_image   FaceBoxesNet.forward_images on the device images that need no shrink / a forward call per
                         image, CUDA events
  detect_ms_per_image    FaceBoxes.detect_images(host images) / N FaceBoxes.__call__, host clock, host images -> box lists
  outputs_ms_per_image   get_all_outputs_images / N get_all_outputs with 16 fixed seeded rects per image, host clock
Medians over the rounds; `spread` is (max - min) / median.  Also printed: the card's name and power limit, detector
launches and host synchronisations per call, and the equality of the two paths' results.  Fails without a GPU."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(ROOT))
import bench  # noqa: E402
from bench_crop import card  # noqa: E402
from bench_frames import alternate, count_syncs, events_ms, wall_ms  # noqa: E402

MIX = ((450, 450), (480, 640), (720, 1080), (1080, 1920), (300, 400))
FACES = 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='1,4,16,64')
    args = ap.parse_args()
    counts = [int(c) for c in args.counts.split(',')]
    if not torch.cuda.is_available():
        raise SystemExit('bench_images.py needs a CUDA device (H100); nothing is measured without one')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    from synergynet_b200 import faceboxes, synthetic
    det = faceboxes.FaceBoxes(weights=synthetic.make_faceboxes_state_dict(0), device='cuda:0')
    net = det.net
    model = bench.build_model(str(dev))
    rng = np.random.default_rng(5)
    out = {'workload': f'uint8 images of sizes drawn from {list(MIX)}, {FACES} seeded rects per image for the outputs rows',
           'card': card(dev), 'counts': {}}
    for n in counts:
        sizes = [MIX[int(k)] for k in rng.integers(0, len(MIX), n)]
        images = [synthetic.make_scene_u8(h, w, 100 + i) for i, (h, w) in enumerate(sizes)]
        dev_images = [torch.from_numpy(im).to(dev) for im in images]
        net_in = [im for im, (h, w) in zip(dev_images, sizes) if h <= 720 and w <= 1080] or dev_images[:1]
        rects = [[[float(x), float(y), float(x + 150), float(y + 180), 0.9]
                  for x, y in rng.uniform([0, 0], [max(w - 300, 1), max(h - 300, 1)], (FACES, 2))] for h, w in sizes]
        net_b = lambda: net.forward_images(net_in)
        net_l = lambda: [net.forward(im) for im in net_in]
        det_b = lambda: det.detect_images(images)
        det_l = lambda: [det(im) for im in images]
        out_b = lambda: model.get_all_outputs_images(images, rects=rects)
        out_l = lambda: [model.get_all_outputs(images[i], rects=rects[i]) for i in range(n)]
        (lb, cb), ll = net_b(), net_l()
        db, dl = det_b(), det_l()
        ob, ol = out_b(), out_l()
        torch.cuda.synchronize()
        pairs = [(np.asarray(a, np.float64), np.asarray(b, np.float64)) for (lg, mg, pg), (lw, mw, pw) in zip(ob, ol)
                 for a, b in (*zip(lg, lw), *zip(mg, mw), *[(np.r_[p[0], p[1]], np.r_[q[0], q[1]]) for p, q in zip(pg, pw)])]
        equal = {'network_bits': all(torch.equal(lb[i], ll[i][0]) and torch.equal(cb[i], ll[i][1]) for i in range(len(net_in))),
                 'detect_lists': db == dl,
                 'outputs_bits': all(np.array_equal(a, b) for a, b in pairs)}
        del ob, ol, pairs
        l0 = net.launch_count
        det_b()
        l1 = net.launch_count
        det_l()
        l2 = net.launch_count
        sb, sl = [0], [0]
        with count_syncs(sb):
            det_b()
        with count_syncs(sl):
            det_l()
        rounds = 7 if n <= 16 else 5
        res = {'sizes': [f'{h}x{w}' for h, w in sizes], 'network_images': len(net_in), 'equal': equal,
               'detector_launches': {'batched': l1 - l0, 'one_image_loop': l2 - l1},
               'detect_host_syncs': {'batched': sb[0], 'one_image_loop': sl[0]},
               'network': alternate(events_ms, net_b, net_l, rounds, len(net_in)),
               'detect': alternate(wall_ms, det_b, det_l, rounds, n),
               'outputs': alternate(wall_ms, out_b, out_l, 5 if n <= 16 else 3, n)}
        out['counts'][str(n)] = res
        print(f'[bench_images] N={n}: ' + json.dumps({k: res[k] for k in ('equal', 'network', 'detect', 'outputs')}), file=sys.stderr)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
