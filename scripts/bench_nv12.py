"""BGR against NV12 frame ingest on bench.py's config 3, and the cost of the inline NV12 conversion per kernel.

    python scripts/bench_nv12.py [--steps 100] [--warmup 10] [--repeats 3] [--kernel-reps 200]

Workload: bench.py config 3 (1920x1080, YOLOv4-csp 640 letterbox + OSNet x1.0, KLT on, detector every K = 5th frame,
200 tracks; synthetic weights, scripted detections fed after the detector ran, real OSNet embeddings).  The frames are
the scene's frames taken to NV12 (oracle/nv12.py); the BGR arms get their cv2 decodes, so all four arms compute the
same tracks (checked: `tracks_equal`).

Four arms, alternated in one call, `repeats` runs each: MOT(pixel_format='BGR') and MOT(pixel_format='NV12'), each fed
frames in pinned host memory and frames resident in device memory.  Host arms read ahead as bench.py's e2e pass does:
MOT.prefetch(frame t + 1) before step t starts that frame's copy on the upload stream under step t, and step t + 1
consumes it (one copy per frame).  A run is `warmup` steps, then `steps` steps timed with CUDA events on the launching
stream.  `h2d_frame_bytes` is counted from the frame copies MOT's uploader made in the timed steps.

Kernel times: CUDA events around `kernel-reps` back-to-back launches of the one-frame entry points on a 1080p frame
(letterbox into the csp-640 input, 200 crops into the OSNet input layout, gray + 0.5x image), each on a BGR and an NV12
FmFrame, median of five sets.  Prints the card name and power limit, then one JSON line.
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


def build_mot(bench, c, scene, total, fmt, first_frame):
    """bench.py's config-3 MOT (same synthetic head gain search) in pixel format `fmt`."""
    from fastmot_b200 import MOT
    args = argparse.Namespace(p5_input=896)
    g0 = float(c.get("synth_head_gain", 1.0))
    for gain in [g0] + [g for g in (0.25, 0.06, 0.015, 0.004) if g < g0]:
        os.environ["FM_SYNTH_HEAD_GAIN"] = str(gain)
        mot = MOT(scene.size, detections_override=bench.det_override(scene, total), pixel_format=fmt,
                  **bench._cfg(c, args))
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
    return mot


def run_arm(mot, frames, W, K):
    """W warm-up steps, K timed steps.  Returns (frames/s, frame H2D bytes per timed step, visible tracks)."""
    mot.reset(1 / 30.)
    for f in frames[:W]:
        mot.step(f)
    host = not torch.is_tensor(frames[0])
    torch.cuda.synchronize()
    b0 = mot._uploader.bytes_copied
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(W, W + K):
        if host and i + 1 < W + K:
            mot.prefetch(frames[i + 1])
        mot.step(frames[i])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / K
    vis = sorted((t.trk_id, tuple(t.tlbr)) for t in mot.visible_tracks())
    return 1000.0 / ms, (mot._uploader.bytes_copied - b0) / K, vis


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
    return round(float(np.median(out)), 2)


def kernel_times(mot_bgr, bgr_frame, nv_frame, scene, reps):
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
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
    s = stream_ptr()
    calls = {
        "letterbox": lambda f: lib.fm_letterbox_preproc(f, in_w, in_h, rx, ry, rw, rh, 1, ptr(inp), s),
        "crops": lambda f: lib.fm_roi_resize_norm(f, ptr(tl), None, n, iw, ih, eng.inp_layout, ptr(crops), s),
        "gray_half": lambda f: lib.fm_gray_half(f, ptr(gray), ptr(small), s),
    }
    frames = {"bgr_us": C.byref(bgr_frame.fm()), "nv12_us": C.byref(nv_frame.fm())}
    out = {}
    for name, call in calls.items():
        out[name] = {}
        for key, f in frames.items():
            _lib.check(call(f), f"{name} {key}")
            out[name][key] = kernel_us(lambda: call(f), reps)
    out["crops"]["n"] = n
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=200)
    args = ap.parse_args()
    import cv2
    import bench
    from bench_multistream import card
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import Frame, nv12_frame
    from oracle.nv12 import bgr_to_nv12
    _lib.require_device()
    print(json.dumps(card()), flush=True)
    c = bench.CONFIGS[3]
    W, K = args.warmup, args.steps
    total = W + K
    scene = bench.make_scene(c, 0)
    nv_host = [bgr_to_nv12(scene.frame(t)) for t in range(total)]
    bgr_host = [cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12) for f in nv_host]
    frames = {
        ("BGR", "host"): [torch.as_tensor(f).pin_memory().numpy() for f in bgr_host],
        ("BGR", "device"): [torch.as_tensor(f).cuda() for f in bgr_host],
        ("NV12", "host"): [torch.as_tensor(f).pin_memory().numpy() for f in nv_host],
        ("NV12", "device"): [torch.as_tensor(f).cuda() for f in nv_host],
    }
    del bgr_host
    mots = {fmt: build_mot(bench, c, scene, total, fmt, frames[(fmt, "device")][0]) for fmt in ("BGR", "NV12")}
    runs = {arm: [] for arm in frames}
    h2d, tracks = {}, {}
    for _ in range(args.repeats):
        for arm, fr in frames.items():
            fps, nbytes, vis = run_arm(mots[arm[0]], fr, W, K)
            runs[arm].append(fps)
            h2d[arm], tracks[arm] = nbytes, vis
    ref = tracks[("BGR", "device")]
    out = {
        "workload": c["workload"], "steps": K, "warmup": W, "repeats": args.repeats,
        "arms": {f"{fmt}/{where}": {"frames_per_s": round(float(np.median(v)), 1), "runs": [round(x, 1) for x in v],
                                     "h2d_frame_bytes": int(h2d[(fmt, where)])}
                 for (fmt, where), v in runs.items()},
        "tracks_equal": all(t == ref for t in tracks.values()),
        "visible_tracks": len(ref),
        "kernels": kernel_times(mots["BGR"], Frame.bgr(frames[("BGR", "device")][0]),
                                nv12_frame(frames[("NV12", "device")][0]), scene, args.kernel_reps),
    }
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
