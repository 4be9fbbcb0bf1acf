"""Aggregate throughput of N camera streams in one process: MultiStreamMOT (one batched YOLO forward and one shared
OSNet batch per detector frame) against N separate MOT objects stepped round-robin, alternated in the same call.

    python scripts/bench_multistream.py [--streams 1,2,4,8] [--steps 200] [--warmup 10] [--repeats 3]

Workload: bench.py config 3 per stream (1080p, YOLOv4-csp 640 letterbox + OSNet x1.0, KLT on, detector every 5th
frame, 200 tracks; synthetic weights, scripted detections fed after the detector ran, real OSNet embeddings).
Frames are resident in device memory.  Prints one JSON line per N with the aggregate frames/s of both arms (median
and spread over the repeats), the detector forward at batch N against N batch-1 forwards, the CUDA-event time per
detector / OSNet forward in each arm, and the device memory of each arm built alone (resident and allocator peak);
the card name and power limit first.
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace as NS

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": plim}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": None}


def forward_ms(eng, reps=20):
    """CUDA-event time of one engine forward (graph replay on the current stream), best of `reps`."""
    eng.warm(2)
    best = float("inf")
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.replay()
        e1.record()
        e1.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,2,4,8")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import bench
    from fastmot_b200 import MOT, MultiStreamMOT, _lib
    from fastmot_b200 import engine as eng_mod
    _lib.require_device()
    c = bench.CONFIGS[3]
    cfg = bench._cfg(c, NS(p5_input=896))
    print(json.dumps(card()), flush=True)

    # the synthetic head gain bench.py settles on for config 3 (candidate count inside key_cap / 2)
    scene0 = bench.make_scene(c, 0)
    f0 = scene0.frame(0)
    for gain in (1.0, 0.25, 0.06, 0.015, 0.004):
        os.environ["FM_SYNTH_HEAD_GAIN"] = str(gain)
        m = MOT(scene0.size, detections_override=bench.det_override(scene0, 1), **cfg)
        m.reset(1 / 30.)
        try:
            m.step(f0)
        except RuntimeError as e:
            if "key_cap" not in str(e):
                raise
            continue
        if m.detector.last_num_candidates <= m.detector.key_cap // 2:
            break
    del m
    torch.cuda.empty_cache()

    T = args.warmup + args.steps
    for N in (int(v) for v in args.streams.split(",")):
        scenes = [bench.make_scene(c, s) for s in range(N)]
        t0 = time.time()
        frames = [[torch.as_tensor(sc.frame(t)).cuda() for sc in scenes] for t in range(T)]
        gen_s = time.time() - t0
        dets = [bench.det_override(sc, T) for sc in scenes]

        def build_ms():
            ms = MultiStreamMOT(scenes[0].size, N, detections_override=lambda s, t: dets[s](t), **cfg)
            ms.extractors[0]._engine(N * c["n"])
            for e in [ms.detector.backend] + list(ms.extractors[0]._engines.values()):
                e.warm(3)
            ms.reset(1 / 30.)
            for t in range(args.warmup):
                ms.step(frames[t])
            return ms

        def build_rr():
            mots = [MOT(scenes[s].size, detections_override=dets[s], **cfg) for s in range(N)]
            for m in mots:
                m.extractors[0]._engine(c["n"])
                for e in [m.detector.backend] + list(m.extractors[0]._engines.values()):
                    e.warm(3)
                m.reset(1 / 30.)
            for t in range(args.warmup):
                for s, m in enumerate(mots):
                    m.step(frames[t][s])
            return mots

        def memory(build):
            """Device memory of one arm built and warmed alone: (resident after the warm-up, allocator peak), both
            above what was allocated before it (the frames)."""
            gc.collect()
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            arm = build()
            torch.cuda.synchronize()
            out = (torch.cuda.memory_allocated() - base, torch.cuda.max_memory_allocated() - base)
            del arm
            gc.collect()
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            return out

        mem_ms, mem_rr = memory(build_ms), memory(build_rr)
        ms, mots = build_ms(), build_rr()

        def run_ms():
            ms.reset(1 / 30.)
            for t in range(args.warmup):
                ms.step(frames[t])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for t in range(args.warmup, T):
                ms.step(frames[t])
            torch.cuda.synchronize()
            return N * args.steps / (time.perf_counter() - t0)

        def run_rr():
            for m in mots:
                m.reset(1 / 30.)
            for t in range(args.warmup):
                for s, m in enumerate(mots):
                    m.step(frames[t][s])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for t in range(args.warmup, T):
                for s, m in enumerate(mots):
                    m.step(frames[t][s])
            torch.cuda.synchronize()
            return N * args.steps / (time.perf_counter() - t0)

        fps_ms, fps_rr = [], []
        for _ in range(args.repeats):           # alternated: both arms see the same machine state
            fps_ms.append(run_ms())
            fps_rr.append(run_rr())

        # stage split: CUDA-event time of each detector / OSNet forward, one profiled pass per arm
        split = {}
        for arm, run in (("multistream", run_ms), ("round_robin", run_rr)):
            prof = eng_mod.enable_profiling()
            run()
            s_ = prof.summary()
            eng_mod._PROF = None
            split[arm] = {"yolo_ms_per_call": round(s_["yolo_ms"] / max(1, s_["yolo_calls"]), 3),
                          "yolo_calls": s_["yolo_calls"],
                          "osnet_ms_per_call": round(s_["osnet_ms"] / max(1, s_["osnet_calls"]), 3),
                          "osnet_calls": s_["osnet_calls"]}
        det_b = forward_ms(ms.detector.backend)
        det_1 = forward_ms(mots[0].detector.backend)
        n_tma = ms.detector.backend.n_tma
        out = {"streams": N, "steps": args.steps, "repeats": args.repeats,
               "multistream_fps": {"median": round(float(np.median(fps_ms)), 1), "min": round(min(fps_ms), 1),
                                   "max": round(max(fps_ms), 1)},
               "round_robin_fps": {"median": round(float(np.median(fps_rr)), 1), "min": round(min(fps_rr), 1),
                                   "max": round(max(fps_rr), 1)},
               "detector_forward_ms": {"batch": round(det_b, 3), "batch1_x_n": round(N * det_1, 3),
                                       "batch1": round(det_1, 3), "convs_on_tma_at_batch": n_tma,
                                       "convs_on_tma_at_1": mots[0].detector.backend.n_tma},
               "stage_split": split,
               "mem_gib": {arm: {"resident": round(m[0] / 2 ** 30, 2), "peak": round(m[1] / 2 ** 30, 2)}
                           for arm, m in (("multistream", mem_ms), ("round_robin", mem_rr))},
               "frame_gen_s": round(gen_s, 1)}
        print(json.dumps(out), flush=True)
        del ms, mots, frames
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
