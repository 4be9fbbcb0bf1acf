"""Step latency of a mixed-size camera group in one process (MultiCameraMOT): all cameras starting together (every
camera's detector frame on the same step) against staggered starts (camera s starts at step floor(s * K / N), so each
step carries about N / K cameras' detector work), alternated in the same call.

    python scripts/bench_multicamera.py [--cameras 4,8] [--steps 200] [--warmup 10] [--repeats 3]

Workload: bench.py config 3 per camera (YOLOv4-csp 640 letterbox + OSNet x1.0, KLT on, detector every K = 5th
frame, up to 200 objects; synthetic weights, scripted detections fed after the detector ran, real OSNet embeddings).
Half the cameras are 1920x1080, half 1280x720; the 720p scenes hold only the objects of the 200-object grid that fall
inside the frame (their track count is printed).  Frames are resident in device memory.  Each `step` is timed with
the host clock and ends in a device synchronise.  The timed window starts `warmup` steps after the last camera
started.  Prints the card name and power limit, then one JSON line per N with the aggregate frames/s and step time
p50 / p99 / max of both schedules (median over the repeats), the step time per detector batch size k, and the CUDA-event
time per YOLO / OSNet forward of each schedule.
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", default="4,8")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import bench
    from bench_multistream import card
    from fastmot_b200 import MOT, MultiCameraMOT, _lib
    from fastmot_b200 import engine as eng_mod
    from fastmot_b200.multicamera import plan_step
    from fastmot_b200.synth import SyntheticScene
    _lib.require_device()
    c = bench.CONFIGS[3]
    cfg = bench._cfg(c, argparse.Namespace(p5_input=896))
    K = c["skip"]
    print(json.dumps(card()), flush=True)

    # the synthetic head gain bench.py settles on for config 3 (candidate count inside key_cap / 2)
    scene0 = bench.make_scene(c, 0)
    for gain in (1.0, 0.25, 0.06, 0.015, 0.004):
        os.environ["FM_SYNTH_HEAD_GAIN"] = str(gain)
        m = MOT(scene0.size, detections_override=bench.det_override(scene0, 1), **cfg)
        m.reset(1 / 30.)
        try:
            m.step(scene0.frame(0))
        except RuntimeError as e:
            if "key_cap" not in str(e):
                raise
            continue
        if m.detector.last_num_candidates <= m.detector.key_cap // 2:
            break
    del m
    torch.cuda.empty_cache()

    for N in (int(v) for v in args.cameras.split(",")):
        sizes = [(1920, 1080)] * (N // 2) + [(1280, 720)] * (N - N // 2)
        schedules = {"aligned": [0] * N, "staggered": [s * K // N for s in range(N)]}
        T = max(max(st) for st in schedules.values()) + args.warmup + args.steps
        scenes = [SyntheticScene(c["n"], size=wh, seed=s, label=0, dropout_frames=(), bounce_radius=16)
                  for s, wh in enumerate(sizes)]
        t0 = time.time()
        frames = [[torch.as_tensor(sc.frame(t)).cuda() for t in range(T)] for sc in scenes]
        gen_s = time.time() - t0
        dets = [bench.det_override(sc, T) for sc in scenes]
        mc = MultiCameraMOT(sizes, detections_override=lambda s, i: dets[s](i), **cfg)
        mc.detector.build_engines()
        mc.extractors[0]._engine(N * c["n"])
        for e in list(mc.detector._engines.values()) + list(mc.extractors[0]._engines.values()):
            e.warm(3)

        def run(starts):
            """Returns the per-step times (ms) of the timed window and each step's detector batch size k."""
            mc.reset(1 / 30.)
            first = max(starts) + args.warmup
            times, ks = [], []
            for t in range(first + args.steps):
                fr = [frames[s][t - st] if t >= st else None for s, st in enumerate(starts)]
                init, detect, _ = plan_step(mc.frame_counts, [f is not None for f in fr], K)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                mc.step(fr)
                torch.cuda.synchronize()
                if t >= first:
                    times.append((time.perf_counter() - t0) * 1e3)
                    ks.append(len(init) + len(detect))
            return np.array(times), np.array(ks)

        for starts in schedules.values():       # untimed: builds the OSNet batch buckets each schedule reaches
            run(starts)
        res = {name: [] for name in schedules}
        for _ in range(args.repeats):           # alternated: both schedules see the same machine state
            for name, starts in schedules.items():
                res[name].append(run(starts))
        out = {"cameras": N, "sizes": [f"{w}x{h}" for w, h in sizes],
               "tracks": [len(mc.trackers[s].tracks) for s in range(N)], "steps": args.steps,
               "repeats": args.repeats, "frame_gen_s": round(gen_s, 1)}
        for name, runs in res.items():
            fps = [N * args.steps / (tm.sum() / 1e3) for tm, _ in runs]
            stat = {q: float(np.median([np.percentile(tm, p) for tm, _ in runs])) for q, p in
                    (("p50", 50), ("p99", 99), ("max", 100))}
            allt, allk = np.concatenate([tm for tm, _ in runs]), np.concatenate([k for _, k in runs])
            by_k = {int(k): {"steps": int((allk == k).sum()), "p50_ms": round(float(np.median(allt[allk == k])), 3),
                             "max_ms": round(float(allt[allk == k].max()), 3)} for k in np.unique(allk)}
            prof = eng_mod.enable_profiling()
            run(schedules[name])
            s_ = prof.summary()
            eng_mod._PROF = None
            out[name] = {"fps": {"median": round(float(np.median(fps)), 1), "min": round(min(fps), 1),
                                 "max": round(max(fps), 1)},
                         "step_ms": {k: round(v, 3) for k, v in stat.items()}, "step_ms_by_k": by_k,
                         "yolo_ms_per_call": round(s_["yolo_ms"] / max(1, s_["yolo_calls"]), 3),
                         "yolo_calls": s_["yolo_calls"],
                         "osnet_ms_per_call": round(s_["osnet_ms"] / max(1, s_["osnet_calls"]), 3),
                         "osnet_calls": s_["osnet_calls"]}
        out["staggered_p99_over_aligned_p99"] = round(out["staggered"]["step_ms"]["p99"] /
                                                      out["aligned"]["step_ms"]["p99"], 3)
        print(json.dumps(out), flush=True)
        del mc, frames
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
