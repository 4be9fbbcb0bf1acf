"""CPU: MultiStreamMOT takes MOT's keyword arguments, so the reference's cfg/mot.json `mot_cfg` passes unchanged."""
import inspect
from types import SimpleNamespace as NS


def _reference_shaped_mot_cfg():
    """The keys of cfg/mot.json's mot_cfg in the reference, with placeholder values."""
    return vars(NS(detector_type='YOLO', detector_frame_skip=5, class_ids=[1], ssd_detector_cfg=NS(),
                   yolo_detector_cfg=NS(), public_detector_cfg=NS(), feature_extractor_cfgs=[NS()], tracker_cfg=NS(),
                   visualizer_cfg=NS()))


def test_multistream_binds_the_reference_mot_cfg():
    from fastmot_b200 import MOT, MultiStreamMOT
    cfg = _reference_shaped_mot_cfg()
    inspect.signature(MOT).bind((1280, 720), **cfg, draw=False)
    inspect.signature(MultiStreamMOT).bind((1280, 720), 4, **cfg, draw=False)


def test_multistream_takes_every_mot_keyword():
    from fastmot_b200 import MOT, MultiStreamMOT
    missing = set(inspect.signature(MOT).parameters) - set(inspect.signature(MultiStreamMOT).parameters)
    assert missing == {'embeddings_tap'}, missing
