"""Frames captured at 1920x1080 and tracked at 1280x720: resize on the host against resize on the GPU, and the time of
the resize kernel itself.

    python scripts/bench_resize.py [--steps 100] [--warmup 10] [--repeats 3] [--kernel-reps 500]

Kernel times: CUDA events around `kernel-reps` back-to-back fm_frame_resize launches, median of five sets, for
1080p BGR -> 720p, 1080p NV12 -> 720p, 4K NV12 -> 1080p (the exact-2x path) and 720p BGR -> 1080p.  Each is reported
beside its compulsory bytes (the source frame read once, the output written once) and the time those bytes take at the
H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth: a computed bound, not a measurement.

End to end: bench.py's config-3 workload (YOLOv4-csp 640 letterbox + OSNet x1.0, KLT on, detector every 5th frame,
200 objects; synthetic weights, scripted detections scaled to 720p fed after the detector ran, real OSNet embeddings)
on 1080p captures tracked at 1280x720.  The captures are the scene's frames taken to NV12 (oracle/nv12.py); the BGR
arms get their cv2 decodes, so the three arms compute the same tracks (checked: `tracks_equal`).  Arms, alternated in
one call, `repeats` runs each:
  host_resize : pinned 1080p BGR host frames, cv2.resize to 720p on the host inside the timed loop, MOT(720p) with
                read-ahead (MOT.prefetch of the next resized frame before each step);
  gpu_resize  : the same host frames into MOT(720p, capture_size=1080p) with read-ahead;
  nv12_device : 1080p NV12 device frames into MOT(720p, capture_size=1080p, pixel_format='NV12').
A run is `warmup` steps, then `steps` steps timed with CUDA events on the launching stream (the host arm's last event
is recorded after its last step was enqueued, so its host resizes are inside the window).  Prints the card name and
power limit, then one JSON line.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet (700 W card)
CAPTURE, TRACK = (1920, 1080), (1280, 720)


def build_mot(bench, c, dets, fmt, capture_size, first_frame):
    """bench.py's config-3 MOT tracked at TRACK (same synthetic head gain search as bench.py)."""
    from fastmot_b200 import MOT
    args = argparse.Namespace(p5_input=896)
    g0 = float(c.get("synth_head_gain", 1.0))
    for gain in [g0] + [g for g in (0.25, 0.06, 0.015, 0.004) if g < g0]:
        os.environ["FM_SYNTH_HEAD_GAIN"] = str(gain)
        mot = MOT(TRACK, detections_override=dets, pixel_format=fmt, capture_size=capture_size, **bench._cfg(c, args))
        try:
            mot.reset(1 / 30.)
            mot.step(first_frame)
        except RuntimeError as e:
            if "key_cap" not in str(e):
                raise
            continue
        if mot.detector.last_num_candidates <= mot.detector.key_cap // 2:
            break
    else:
        raise RuntimeError("no synthetic head gain keeps the candidate count inside key_cap")
    mot.extractors[0]._engine(c["n"])
    for e in [mot.detector.backend] + list(mot.extractors[0]._engines.values()):
        e.warm(3)
    return mot, gain


def scaled_dets(bench, scene, total):
    """bench.det_override's scripted boxes, scaled from CAPTURE to TRACK."""
    base = bench.det_override(scene, total)
    k = np.array([TRACK[0] / CAPTURE[0], TRACK[1] / CAPTURE[1]] * 2)

    def f(t):
        d = base(t)
        d.tlbr = d.tlbr * k
        return d
    return f


def run_arm(mot, frames, W, K, host_resize=False):
    """W warm-up steps, K timed steps.  Returns (frames/s, visible tracks).  host_resize: every frame goes through
    cv2.resize(frame, TRACK) on the host first."""
    import cv2
    prep = (lambda f: cv2.resize(f, TRACK)) if host_resize else (lambda f: f)
    mot.reset(1 / 30.)
    for f in frames[:W]:
        mot.step(prep(f))
    host = not torch.is_tensor(frames[0])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    nxt = prep(frames[W])
    for i in range(W, W + K):
        cur = nxt
        if i + 1 < W + K:
            nxt = prep(frames[i + 1])
            if host:
                mot.prefetch(nxt)
        mot.step(cur)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    vis = sorted((t.trk_id, tuple(t.tlbr)) for t in mot.visible_tracks())
    return 1000.0 / ms, vis


def kernel_us(fn, reps):
    """Median over five sets of the CUDA-event time per call of `reps` back-to-back calls of fn()."""
    for _ in range(3):
        fn()
    out = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1000.0 / reps)
    return float(np.median(out))


def kernel_times(reps):
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import Frame, nv12_frame, ptr, stream_ptr
    lib = _lib.load()
    rng = np.random.default_rng(0)
    cases = [("1080p BGR -> 720p", "BGR", (1920, 1080), (1280, 720)),
             ("1080p NV12 -> 720p", "NV12", (1920, 1080), (1280, 720)),
             ("4K NV12 -> 1080p", "NV12", (3840, 2160), (1920, 1080)),
             ("720p BGR -> 1080p", "BGR", (1280, 720), (1920, 1080))]
    out = []
    for name, fmt, (sw, sh), (dw, dh) in cases:
        shape = (sh, sw, 3) if fmt == "BGR" else (3 * sh // 2, sw)
        src = torch.as_tensor(rng.integers(0, 256, shape, dtype=np.uint8)).cuda()
        f = Frame.bgr(src) if fmt == "BGR" else nv12_frame(src)
        dst = torch.empty((dh, dw, 3), dtype=torch.uint8, device="cuda")
        fm, s = C.byref(f.fm()), stream_ptr()
        _lib.check(lib.fm_frame_resize(fm, ptr(dst), dw, dh, s), name)
        us = kernel_us(lambda: lib.fm_frame_resize(fm, ptr(dst), dw, dh, s), reps)
        nbytes = src.numel() + dst.numel()
        bound_us = nbytes / HBM_BYTES_PER_S * 1e6
        out.append({"case": name, "kernel_us": round(us, 2), "read_bytes": src.numel(), "write_bytes": dst.numel(),
                    "hbm_bound_us": round(bound_us, 2), "frac_of_hbm_bound": round(bound_us / us, 3)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=500)
    args = ap.parse_args()
    import cv2
    import bench
    from bench_multistream import card
    from fastmot_b200 import _lib
    from oracle.nv12 import bgr_to_nv12
    _lib.require_device()
    print(json.dumps(card()), flush=True)
    kernels = kernel_times(args.kernel_reps)
    c = bench.CONFIGS[3]
    W, K = args.warmup, args.steps
    total = W + K
    scene = bench.make_scene(c, 0)
    assert tuple(scene.size) == CAPTURE
    nv_host = [bgr_to_nv12(scene.frame(t)) for t in range(total)]
    bgr_pinned = [torch.as_tensor(cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12)).pin_memory().numpy() for f in nv_host]
    nv_dev = [torch.as_tensor(f).cuda() for f in nv_host]
    del nv_host
    dets = scaled_dets(bench, scene, total)
    mots, gains = {}, {}
    mots["host_resize"], gains["host_resize"] = build_mot(bench, c, dets, "BGR", None, cv2.resize(bgr_pinned[0], TRACK))
    mots["gpu_resize"], gains["gpu_resize"] = build_mot(bench, c, dets, "BGR", CAPTURE, bgr_pinned[0])
    mots["nv12_device"], gains["nv12_device"] = build_mot(bench, c, dets, "NV12", CAPTURE, nv_dev[0])
    frames = {"host_resize": bgr_pinned, "gpu_resize": bgr_pinned, "nv12_device": nv_dev}
    runs = {arm: [] for arm in frames}
    tracks = {}
    for _ in range(args.repeats):
        for arm, fr in frames.items():
            fps, vis = run_arm(mots[arm], fr, W, K, host_resize=arm == "host_resize")
            runs[arm].append(fps)
            tracks[arm] = vis
    ref = tracks["host_resize"]
    out = {
        "workload": c["workload"] + f"; captured at {CAPTURE[0]}x{CAPTURE[1]}, tracked at {TRACK[0]}x{TRACK[1]}",
        "steps": K, "warmup": W, "repeats": args.repeats, "synth_head_gain": gains,
        "kernels": kernels,
        "arms": {arm: {"frames_per_s": round(float(np.median(v)), 1), "min": round(min(v), 1),
                       "max": round(max(v), 1), "runs": [round(x, 1) for x in v]} for arm, v in runs.items()},
        "tracks_equal": all(t == ref for t in tracks.values()),
        "visible_tracks": len(ref),
    }
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
