"""Frame-batch measurement: the batched path against a loop of the one-image calls on the same frames, in one command.
    python scripts/bench_frames.py [--counts 1,4,16,64] > frames_bench.json

Frames: seeded synthetic.make_scene_u8 scenes at 720 x 1080 (16 distinct scenes, frame i = scene i mod 16); detector
weights: synthetic.make_faceboxes_state_dict(0); backbone: bench.py's seeded mobilenet_v2.  For every frame count N, with
every shape warmed up first and the two paths alternating round by round:
  network_ms_per_frame   FaceBoxesNet.forward_batch on the N-frame device stack / N forward calls, CUDA events
  detect_ms_per_frame    FaceBoxes.detect_batch(host frames) / N FaceBoxes.__call__, host clock, host frames -> box lists
  outputs_ms_per_frame   get_all_outputs_batch / N get_all_outputs with 16 fixed seeded rects per frame (the synthetic
                         detector's boxes are not face-like), host clock, host frames -> landmarks, dense meshes, poses
A timed window holds at least 16 frames of work (16 // N repeats of the call).  Medians over the rounds; `spread` is (max - min) / median of the rounds.  Also printed: the card's name and power limit,
detector launches and host synchronisations per call as counted here, and the equality of the two paths' results at the
timed sizes.  When batching does not lower the network time per frame at N = 16, the per-launch times of both paths are
added (differences of runs stopped after consecutive launches).  Fails without a GPU."""
import argparse
import contextlib
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from bench_crop import card  # noqa: E402

H, W, FACES = 720, 1080, 16


@contextlib.contextmanager
def count_syncs(counter):
    """Count the host synchronisations torch makes: .item(), .cpu(), .tolist(), stream / device synchronize."""
    saved = {}

    def wrap(owner, name):
        fn = getattr(owner, name)
        saved[(owner, name)] = fn

        def counted(*a, **k):
            if owner is not torch.Tensor or a[0].is_cuda:
                counter[0] += 1
            return fn(*a, **k)
        setattr(owner, name, counted)
    for owner, name in ((torch.Tensor, 'item'), (torch.Tensor, 'cpu'), (torch.Tensor, 'tolist'), (torch.cuda.Stream, 'synchronize'),
                        (torch.cuda, 'synchronize')):
        wrap(owner, name)
    try:
        yield
    finally:
        for (owner, name), fn in saved.items():
            setattr(owner, name, fn)


def events_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def wall_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def alternate(timer, batched, looped, rounds, n):
    reps = max(1, 16 // n)                     # a timed window holds at least 16 frames of work
    tb, tl = [], []
    for _ in range(rounds):
        tb.append(timer(lambda: [batched() for _ in range(reps)]) / (n * reps))
        tl.append(timer(lambda: [looped() for _ in range(reps)]) / (n * reps))
    stat = lambda t: {'ms_per_frame': statistics.median(t), 'spread': (max(t) - min(t)) / statistics.median(t), 'rounds': len(t)}
    return {'batched': stat(tb), 'one_image_loop': stat(tl), 'ratio_loop_over_batched': statistics.median(tl) / statistics.median(tb)}


def per_launch(net, stack, one):
    """ms of every launch, batched (per call) and one image: differences of runs stopped after consecutive launches."""
    def cumulative(fn):
        out = []
        for s in range(39):
            fn(s)
            out.append(min(events_ms(lambda: fn(s)) for _ in range(3)))
        return out
    cb = cumulative(lambda s: net.debug_forward_batch_until(stack, s))
    c1 = cumulative(lambda s: net.debug_forward_until(one, s))
    diff = lambda c: [c[0]] + [c[i] - c[i - 1] for i in range(1, 39)]
    return {'what': 'stage s minus stage s-1 of the debug stops (each includes its device-to-device copy of the stage output)',
            'batched_ms': diff(cb), 'one_image_ms': diff(c1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--counts', default='1,4,16,64')
    args = ap.parse_args()
    counts = [int(c) for c in args.counts.split(',')]
    if not torch.cuda.is_available():
        raise SystemExit('bench_frames.py needs a CUDA device (H100); nothing is measured without one')
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    from synergynet_b200 import faceboxes, synthetic
    scenes = [synthetic.make_scene_u8(H, W, s) for s in range(16)]
    det = faceboxes.FaceBoxes(weights=synthetic.make_faceboxes_state_dict(0), device='cuda:0')
    net = det.net
    model = bench.build_model(str(dev))
    rng = np.random.default_rng(3)
    out = {'workload': f'{H}x{W}x3 uint8 frames, {FACES} seeded rects per frame for the outputs rows', 'card': card(dev), 'counts': {}}
    for n in counts:
        frames = np.stack([scenes[i % 16] for i in range(n)])
        stack = torch.from_numpy(frames).to(dev)
        rects = [[[float(x), float(y), float(x + 150), float(y + 180), 0.9] for x, y in rng.uniform([0, 0], [W - 300, H - 300], (FACES, 2))]
                 for _ in range(n)]
        net_b = lambda: net.forward_batch(stack)
        net_l = lambda: [net.forward(stack[i]) for i in range(n)]
        det_b = lambda: det.detect_batch(frames)
        det_l = lambda: [det(frames[i]) for i in range(n)]
        out_b = lambda: model.get_all_outputs_batch(frames, rects=rects)
        out_l = lambda: [model.get_all_outputs(frames[i], rects=rects[i]) for i in range(n)]
        # warm-up of every shape, and the equality of the two paths at this size
        (lb, cb), ll = net_b(), net_l()
        db, dl = det_b(), det_l()
        ob, ol = out_b(), out_l()
        torch.cuda.synchronize()
        pairs = [(np.asarray(a, np.float64), np.asarray(b, np.float64)) for (lg, mg, pg), (lw, mw, pw) in zip(ob, ol)
                 for a, b in (*zip(lg, lw), *zip(mg, mw), *[(np.r_[p[0], p[1]], np.r_[q[0], q[1]]) for p, q in zip(pg, pw)])]
        equal = {'network_bits': all(torch.equal(lb[i], ll[i][0]) and torch.equal(cb[i], ll[i][1]) for i in range(n)),
                 'detect_lists': db == dl,
                 'outputs_faces': [len(pairs) // 3, sum(len(t[0]) for t in ol)],
                 'outputs_bits': all(np.array_equal(a, b) for a, b in pairs),
                 'outputs_max_rel_diff': max(float(np.abs(a - b).max() / np.abs(b).max()) for a, b in pairs)}
        del ob, ol, pairs
        l0 = net.launch_count
        net_b()
        l1 = net.launch_count
        net_l()
        l2 = net.launch_count
        sb, sl = [0], [0]
        with count_syncs(sb):
            det_b()
        with count_syncs(sl):
            det_l()
        rounds = 7 if n <= 16 else 5
        res = {'equal': equal,
               'detector_launches': {'batched': l1 - l0, 'one_image_loop': l2 - l1},
               'detect_host_syncs': {'batched': sb[0], 'one_image_loop': sl[0]},
               'network': alternate(events_ms, net_b, net_l, rounds, n),
               'detect': alternate(wall_ms, det_b, det_l, rounds, n),
               'outputs': alternate(wall_ms, out_b, out_l, 5 if n <= 16 else 3, n)}
        if n == 16 and res['network']['ratio_loop_over_batched'] <= 1.0:
            res['per_launch'] = per_launch(net, stack, stack[0])
        out['counts'][str(n)] = res
        print(f'[bench_frames] N={n}: ' + json.dumps({k: res[k] for k in ('equal', 'network', 'detect', 'outputs')}), file=sys.stderr)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
