"""Frame ingest in every pixel format on bench.py's config 3, and the cost of reading each format in place per kernel.

    python scripts/bench_pixfmt.py [--steps 100] [--warmup 10] [--repeats 3] [--kernel-reps 200]

Workload: bench.py config 3 (1920x1080, YOLOv4-csp 640 letterbox + OSNet x1.0, KLT on, detector every K = 5th frame,
200 tracks; synthetic weights, scripted detections fed after the detector ran, real OSNet embeddings), as in
scripts/bench_nv12.py.  The scene's frames are encoded with cv2 to NV12, I420, YUY2 and BGRx (oracle/pixfmt.py); the BGR
arms get the scene's BGR frames.  The 4:2:0 and 4:2:2 encodes lose chroma, so their tracks are compared against the BGR
path on their own cv2 decode by the tests, not here; `visible_tracks` is reported per arm.

Ten arms, alternated in one call, `repeats` runs each: MOT(pixel_format=fmt) for each of the five formats, fed frames in
pinned host memory (read ahead with MOT.prefetch, as bench.py's e2e pass does) and frames resident in device memory.  A
run is `warmup` steps, then `steps` steps timed with CUDA events on the launching stream.  `h2d_frame_bytes` is counted
from the frame copies MOT's uploader made in the timed steps (1080p: BGR 6 220 800, BGRx 8 294 400, YUY2 4 147 200,
NV12 and I420 3 110 400).

Kernel times: CUDA events around `kernel-reps` back-to-back launches of the one-frame entry points on a 1080p frame of
each format (letterbox into the csp-640 input, 200 crops into the OSNet input layout, gray + 0.5x image, fm_frame_resize
to 1280x720), median of five sets.  `host_cvtcolor_us` is, for scale only, the CPU time of the cv2.cvtColor decode a
caller would otherwise run per frame on the launching thread (median of 50 calls; cv2's own thread count).  Prints the
card name and power limit, then one JSON line.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

FMTS = ("BGR", "NV12", "I420", "YUY2", "BGRX")


def encode(bgr, fmt):
    from oracle import pixfmt
    from oracle.nv12 import bgr_to_nv12
    if fmt == "BGR":
        return bgr
    if fmt == "NV12":
        return bgr_to_nv12(bgr)
    return pixfmt.DECODES[fmt][2](bgr)


def kernel_times(mot_bgr, frames, scene, reps):
    """{kernel: {fmt: us per call}} on the device Frames `frames` (fmt -> Frame)."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    from bench_nv12 import kernel_us
    lib = _lib.load()
    W, H = scene.size
    det = mot_bgr.detector
    in_w, in_h = det.input_wh
    rx, ry, rw, rh = det.roi
    inp = torch.empty_like(det.inp)
    eng = mot_bgr.extractors[0]._engine(200)
    _, ih, iw = mot_bgr.extractors[0].model.INPUT_SHAPE
    crops = torch.zeros_like(eng.inp)
    tl = torch.as_tensor(np.ascontiguousarray(scene.detections(0)[0][:200])).cuda()
    n = len(tl)
    gray = torch.empty(H, W, dtype=torch.uint8, device="cuda")
    small = torch.empty(H // 2, W // 2, dtype=torch.uint8, device="cuda")
    resized = torch.empty(720, 1280, 3, dtype=torch.uint8, device="cuda")
    s = stream_ptr()
    calls = {
        "letterbox": lambda f: lib.fm_letterbox_preproc(f, in_w, in_h, rx, ry, rw, rh, 1, ptr(inp), s),
        "crops": lambda f: lib.fm_roi_resize_norm(f, ptr(tl), None, n, iw, ih, eng.inp_layout, ptr(crops), s),
        "gray_half": lambda f: lib.fm_gray_half(f, ptr(gray), ptr(small), s),
        "frame_resize_720p": lambda f: lib.fm_frame_resize(f, ptr(resized), 1280, 720, s),
    }
    out = {}
    for name, call in calls.items():
        out[name] = {}
        for fmt, fr in frames.items():
            f = C.byref(fr.fm())
            _lib.check(call(f), f"{name} {fmt}")
            out[name][fmt] = kernel_us(lambda: call(f), reps)
    out["crops"]["n"] = n
    return out


def host_cvtcolor_us(raw):
    """Median CPU time of cv2.cvtColor(frame, decode code) per 1080p frame of each raw format."""
    from oracle.pixfmt import cv2_decode
    out = {}
    for fmt, f in raw.items():
        if fmt == "BGR":
            continue
        ts = []
        for _ in range(50):
            t0 = time.perf_counter()
            cv2_decode(f, fmt)
            ts.append(time.perf_counter() - t0)
        out[fmt] = round(float(np.median(ts)) * 1e6, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=200)
    args = ap.parse_args()
    import bench
    from bench_multistream import card
    from bench_nv12 import build_mot, run_arm
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import pixel_frame
    _lib.require_device()
    print(json.dumps(card()), flush=True)
    c = bench.CONFIGS[3]
    W, K = args.warmup, args.steps
    total = W + K
    scene = bench.make_scene(c, 0)
    bgr = [scene.frame(t) for t in range(total)]
    frames = {}
    for fmt in FMTS:
        raw = [encode(f, fmt) for f in bgr]
        frames[(fmt, "host")] = [torch.as_tensor(f).pin_memory().numpy() for f in raw]
        frames[(fmt, "device")] = [torch.as_tensor(f).cuda() for f in raw]
    first = {fmt: frames[(fmt, "host")][0] for fmt in FMTS}
    del bgr
    mots = {fmt: build_mot(bench, c, scene, total, fmt, frames[(fmt, "device")][0]) for fmt in FMTS}
    runs = {arm: [] for arm in frames}
    h2d, tracks = {}, {}
    for _ in range(args.repeats):
        for arm, fr in frames.items():
            fps, nbytes, vis = run_arm(mots[arm[0]], fr, W, K)
            runs[arm].append(fps)
            h2d[arm], tracks[arm] = nbytes, vis
    out = {
        "workload": c["workload"], "steps": K, "warmup": W, "repeats": args.repeats,
        "arms": {f"{fmt}/{where}": {"frames_per_s": round(float(np.median(v)), 1), "runs": [round(x, 1) for x in v],
                                     "h2d_frame_bytes": int(h2d[(fmt, where)]),
                                     "visible_tracks": len(tracks[(fmt, where)])}
                 for (fmt, where), v in runs.items()},
        "host_equals_device": all(tracks[(fmt, "host")] == tracks[(fmt, "device")] for fmt in FMTS),
        "kernels": kernel_times(mots["BGR"], {fmt: pixel_frame(frames[(fmt, "device")][0], fmt) for fmt in FMTS},
                                scene, args.kernel_reps),
        "host_cvtcolor_us": host_cvtcolor_us(first),
    }
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
