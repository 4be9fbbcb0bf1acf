"""Track record (API of fastmot/track.py:129-225) whose heavy state lives in device pools.

Host side keeps what the reference keeps as Python scalars/containers (ids, age, hits, box history);
Kalman state, running-average feature and keypoints live in slot-indexed device tensors (`TrackPool`)
and are fetched lazily through the same attribute names (`state`, `avg_feat()`, `keypoints`).
"""
from collections import deque

import numpy as np

from .models.label import get_label_name


class AverageFeature:
    """Running mean of embeddings (fastmot/track.py:91-126); arrays live in the pool."""

    def __init__(self, pool, slot):
        self._pool = pool
        self._slot = slot
        self.count = 0

    def __call__(self):
        if self.count == 0:
            return None
        return self._pool.fetch_feature(self._slot, avg=True)

    @property
    def sum(self):
        return None if self.count == 0 else self._pool.fetch_feature(self._slot, avg=False)

    @property
    def avg(self):
        return self()

    def is_valid(self):
        return self.count > 0


class Track:
    def __init__(self, trk_id, frame_id, tlbr, pool, label, confirm_hits=1, buffer_size=30, slot=None):
        # the id comes from the owning MultiTracker: every tracker numbers its own tracks from 1
        self.trk_id = trk_id
        self._pool = pool
        self.slot = pool.acquire() if slot is None else slot
        self.start_frame = frame_id
        self.frame_ids = deque([frame_id], maxlen=buffer_size)
        self.bboxes = deque([tlbr], maxlen=buffer_size)
        self.confirm_hits = confirm_hits
        self.label = label

        self.age = 0
        self.hits = 0
        self.avg_feat = AverageFeature(pool, self.slot)

    def __str__(self):
        x = (self.tlbr[0] + self.tlbr[2]) / 2
        y = (self.tlbr[1] + self.tlbr[3]) / 2
        return f'{get_label_name(self.label):<10} {self.trk_id:>3} at ({int(x):>4}, {int(y):>4})'

    __repr__ = __str__

    def __len__(self):
        return self.end_frame - self.start_frame

    def __lt__(self, other):
        # closer to the image plane is greater (fastmot/track.py:160-162)
        return (self.tlbr[-1], -self.age) < (other.tlbr[-1], -other.age)

    @property
    def tlbr(self):
        return self.bboxes[-1]

    @property
    def end_frame(self):
        return self.frame_ids[-1]

    @property
    def active(self):
        return self.age < 2

    @property
    def confirmed(self):
        return self.hits >= self.confirm_hits

    # ---- device-backed attributes (lazy D2H; synchronises) ----
    @property
    def state(self):
        return self._pool.fetch_state(self.slot)

    @property
    def inlier_ratio(self):
        return self._pool.fetch_scalar('inlier_ratio', self.slot)

    @property
    def keypoints(self):
        return self._pool.fetch_keypoints(self.slot, prev=False)

    @property
    def prev_keypoints(self):
        return self._pool.fetch_keypoints(self.slot, prev=True)

    @property
    def last_feat(self):
        return self._pool.fetch_last_feat(self.slot) if self.avg_feat.count else None

    # ---- host bookkeeping (device side is updated by batched kernels in MultiTracker) ----
    def update(self, tlbr):
        self.bboxes.append(tlbr)

    def add_detection(self, frame_id, tlbr, is_valid=True):
        self.frame_ids.append(frame_id)
        self.bboxes.append(tlbr)
        if is_valid:
            self.avg_feat.count += 1
        self.age = 0
        self.hits += 1

    def reinstate(self, frame_id, tlbr):
        self.start_frame = frame_id
        self.frame_ids.append(frame_id)
        self.bboxes.append(tlbr)
        self.avg_feat.count += 1
        self.age = 0

    def mark_missed(self):
        self.age += 1
