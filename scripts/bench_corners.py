"""Cost of corner re-detection in large track boxes: the KLT stage with 0, 1 and 4 large textured boxes.

    python scripts/bench_corners.py [--steps 30] [--warmup 5] [--out DIR]

Workload: 1920x1080, SyntheticScene's 200 ordinary objects plus 0, 1 or 4 large boxes (640x640 or 1000x1000) of
`smooth_texture` at factor 10, 6 or 3; the smaller the factor, the finer the texture and the more corner candidates
(local maxima above the quality threshold) a box holds, from about 4 500 to 43 000 per box.  Default flow_cfg.

Each step is MultiTracker.compute_flow + apply_kalman on the same frame pair (the call the tracker makes every frame)
after the track pool's keypoint counts are cleared, so every track re-detects its corners in every step: the worst
case of the stage.  Host clock from before compute_flow to a device synchronise after apply_kalman; the clearing
memset runs before the clock starts.  `warmup` untimed steps first.  Per arm: mean and min step time, the largest
candidate count of a visible crop (counted with OpenCV on the host), and for comparison the host time of
cv2.goodFeaturesToTrack on each large box (default setting, mean of 3), a CPU figure that says nothing about the GPU.
Prints the card name and power limit, then one JSON line (also written to DIR/bench_corners.json with --out).
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SIZES = (640, 1000)
FACTORS = (10, 6, 3)
# top-left corners of the large boxes, nearest (lowest bottom edge) last
ORIGINS = {640: [(40, 20), (680, 60), (1240, 100), (360, 420)], 1000: [(0, 0), (900, 20), (400, 40), (880, 70)]}


def scene_frame(scene, n_big, side, factor):
    from fastmot_b200.synth import smooth_texture
    rng = np.random.default_rng(1000 * side + factor)
    frames = []
    tex = [smooth_texture(rng, side, side, factor) for _ in range(n_big)]
    for t in (0, 1):
        f = scene.frame(t)
        for i in range(n_big):
            x, y = ORIGINS[side][i]
            f[y:y + side, x:x + side] = tex[i]
        frames.append(f)
    tl, lb, cf, _ = scene.detections(0)
    big = np.array([(x, y, x + side - 1, y + side - 1) for x, y in ORIGINS[side][:n_big]], np.float64).reshape(-1, 4)
    return frames, np.concatenate([tl, big]), np.concatenate([lb, np.zeros(n_big, lb.dtype)]), \
        np.concatenate([cf, np.full(n_big, 0.9)])


def _dets(tlbr, labels, conf):
    dt = np.dtype([('tlbr', float, 4), ('label', int), ('conf', float)], align=True)
    arr = np.zeros(len(tlbr), dt)
    arr['tlbr'], arr['label'], arr['conf'] = tlbr, labels, conf
    return arr.view(np.recarray)


def run_arm(scene, n_big, side, factor, steps, warmup):
    import cv2
    from fastmot_b200 import MultiTracker
    from oracle.run import default_tracker_cfg
    from test_corner_candidates_cpu import box_candidates
    frames, tlbr, labels, conf = scene_frame(scene, n_big, side, factor)
    trk = MultiTracker(scene.size, 'cosine', **default_tracker_cfg())
    trk.reset(1 / 30)
    trk.init(frames[0], _dets(tlbr, labels, conf))
    times = []
    for i in range(warmup + steps):
        trk.pool.kp_count.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        trk.compute_flow(frames[1])
        trk.apply_kalman()
        torch.cuda.synchronize()
        if i >= warmup:
            times.append(time.perf_counter() - t0)
    cands = box_candidates(frames[0], tlbr)
    gray = cv2.cvtColor(frames[0], cv2.COLOR_BGR2GRAY)
    cpu = []
    for x0, y0, x1, y1 in tlbr[len(tlbr) - n_big:].astype(int):
        crop = gray[y0:y1 + 1, x0:x1 + 1]
        md = max(round(np.sqrt(crop.size) * 0.06), 1)
        t0 = time.perf_counter()
        for _ in range(3):
            cv2.goodFeaturesToTrack(crop, 1000, 0.06, md, blockSize=3)
        cpu.append((time.perf_counter() - t0) / 3 * 1e3)
    return dict(n_big=n_big, side=side, factor=factor, tracks=len(tlbr),
                mean_ms=float(np.mean(times) * 1e3), min_ms=float(np.min(times) * 1e3),
                max_candidates=int(max(cands)), big_candidates=[int(c) for c in cands[len(cands) - n_big:]],
                cv2_gftt_ms_per_box=[round(c, 2) for c in cpu])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_corners.py measures the GPU"
    import subprocess
    from fastmot_b200.synth import SyntheticScene
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    scene = SyntheticScene(200, seed=0, label=0, dropout_frames=())
    arms = [(0, 640, 10)] + [(n, s, f) for s in SIZES for f in FACTORS for n in (1, 4)]
    rows = []
    for n, s, f in arms:
        r = run_arm(scene, n, s, f, args.steps, args.warmup)
        rows.append(r)
        print(f"{n} x {s}^2 factor {f}: {r['mean_ms']:.3f} ms (min {r['min_ms']:.3f}), "
              f"candidates {r['big_candidates']}, cv2 {r['cv2_gftt_ms_per_box']} ms/box", flush=True)
    out = dict(card=card, steps=args.steps, warmup=args.warmup, arms=rows)
    print(json.dumps(out))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_corners.json"), "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
