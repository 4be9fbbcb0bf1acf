"""CPU: MultiCameraMOT takes MOT's keyword arguments, and its per-step schedule (which cameras init, detect, track or
are absent) follows MOT's cadence on each camera's own frames."""
import inspect

from test_multistream_cpu import _reference_shaped_mot_cfg


def test_multicamera_binds_the_reference_mot_cfg():
    from fastmot_b200 import MOT, MultiCameraMOT
    cfg = _reference_shaped_mot_cfg()
    inspect.signature(MultiCameraMOT).bind([(1920, 1080), (1280, 720), (1024, 768)], **cfg, draw=False)
    missing = set(inspect.signature(MOT).parameters) - set(inspect.signature(MultiCameraMOT).parameters)
    assert missing == {'embeddings_tap', 'size'}, missing


def test_plan_step_follows_each_cameras_own_frame_count():
    from fastmot_b200.multicamera import plan_step
    # camera 0 at local frame 0, 1 on a detector frame, 2 between detector frames, 3 absent, 4 on a detector frame
    assert plan_step([0, 10, 7, 5, 5], [True, True, True, False, True], 5) == ([0], [1, 4], [2])
    assert plan_step([0, 0], [False, False], 5) == ([], [], [])
    assert plan_step([3, 4], [True, True], 1) == ([], [0, 1], [])


def schedule(detector_frame_skip=5):
    """The schedule of tests/test_gpu_multicamera.py: camera 0 from step 0 to 21, camera 1 from step 2 (reset before
    step 14, no frame at step 16), camera 2 from step 3 (no frame at steps 9 and 10).  Returns, per step, the
    (init, detect, track) cameras."""
    from fastmot_b200.multicamera import plan_step
    counts, out = [0, 0, 0], []
    for t in range(24):
        if t == 14:
            counts[1] = 0
        present = [t < 22, t >= 2 and t != 16, t >= 3 and t not in (9, 10)]
        plan = plan_step(counts, present, detector_frame_skip)
        for s in sum(plan, []):
            counts[s] += 1
        out.append(plan)
    return out


def test_staggered_schedule_reaches_three_batch_sizes():
    plans = schedule()
    ks = [len(i) + len(d) for i, d, _ in plans]
    assert {k for k in ks if k} == {1, 2, 3}, ks
    assert plans[14][0] == [1]                      # the reconnect re-initialises camera 1
    assert plans[15][1] == [0, 2] and plans[20][1] == [0, 1, 2]
    assert plans[8] == ([], [2], [0, 1])            # camera 2 alone on a detector frame: slot 0 of the batch
    assert all(2 not in sum(plans[t], []) for t in (9, 10))
