"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/seq_flow_cfg.npz by running the UNMODIFIED reference MultiTracker
(imported through oracle/refshim.py) with flow_cfg settings other than cfg/mot.json's: other frame sizes, optical-flow
scales and goodFeaturesToTrack settings.  tests/test_flow_cfg_oracle.py and tests/test_gpu_flow_cfg.py replay the
cases below.  Run where the reference tree is present:  python -m oracle.flow_cfg_goldens
"""
import os
import sys
from types import SimpleNamespace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fastmot_b200.synth import SyntheticScene  # noqa: E402
from oracle.ref_run import run_reference_tracker  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

# (name, scene kwargs, frames, flow_cfg overrides, obj_feat_params overrides)
FLOW_CFG_CASES = [
    ('odd_default', dict(n_objects=90, size=(1173, 880), seed=31), 25, {}, {}),
    ('anisotropic_bs5_unlimited', dict(n_objects=60, seed=32), 25,
     dict(opt_flow_scale_factor=(0.4, 0.6)), dict(maxCorners=0, blockSize=5)),
    ('full_scale_harris_g5', dict(n_objects=110, size=(1281, 721), seed=33), 25,
     dict(opt_flow_scale_factor=(1.0, 1.0), bg_feat_scale_factor=(0.15, 0.15)),
     dict(useHarrisDetector=True, k=0.04, gradientSize=5)),
]


def flow_cfg_namespace(base, flow_over, feat_over):
    """A copy of the SimpleNamespace flow_cfg `base` with the overrides applied (obj_feat_params copied too)."""
    cfg = SimpleNamespace(**vars(base))
    for k, v in flow_over.items():
        setattr(cfg, k, v)
    cfg.obj_feat_params = SimpleNamespace(**dict(vars(base.obj_feat_params), **feat_over))
    return cfg


def flow_cfg_golden():
    """Visible ids / boxes, KLT ids / boxes and H per frame of the reference MultiTracker for FLOW_CFG_CASES."""
    from oracle.refshim import reference_config
    base = reference_config().mot_cfg.tracker_cfg.flow_cfg
    rec = {}
    for i, (name, scene_kw, n_frames, flow_over, feat_over) in enumerate(FLOW_CFG_CASES):
        def capture(t, trk, phase, i=i):
            if phase == 'flow':
                ids = np.array(list(trk.klt_bboxes.keys()), np.int64)
                rec[f'c{i}_klt_ids_{t}'] = ids
                rec[f'c{i}_klt_tlbr_{t}'] = np.array([trk.klt_bboxes[k] for k in ids], np.float64).reshape(-1, 4)
                rec[f'c{i}_H_{t}'] = np.zeros((0,)) if trk.homography is None else np.array(trk.homography, np.float64)
        cfg = flow_cfg_namespace(base, flow_over, feat_over)
        out, trk = run_reference_tracker(SyntheticScene(**scene_kw), n_frames, capture=capture,
                                         tracker_kwargs={'flow_cfg': cfg})
        for t, o in enumerate(out):
            rec[f'c{i}_vis_ids_{t}'] = o['ids']
            rec[f'c{i}_vis_tlbr_{t}'] = o['tlbr']
        rec[f'c{i}_name'] = np.array(name)
        print(name, 'frames', n_frames, 'visible at the end', len(out[-1]['ids']),
              'klt boxes at the end', len(rec[f'c{i}_klt_ids_{n_frames - 1}']))
    rec['n_cases'] = np.int64(len(FLOW_CFG_CASES))
    np.savez_compressed(os.path.join(OUT, 'seq_flow_cfg.npz'), **rec)


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    flow_cfg_golden()
