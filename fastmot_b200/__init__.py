"""fastmot_b200 — H100-native implementation of the FastMOT per-frame hot path.

Public names mirror fastmot/__init__.py:1-7 of the reference (VideoIO is out of scope: SURVEY.md §2.1 row 13).
"""
from .track import Track
from .kalman_filter import KalmanFilter, MeasType
from .flow import Flow
from .tracker import MultiTracker, DeviceEmbeddings
from .detector import YOLODetector, PublicDetector, DET_DTYPE
from .feature_extractor import FeatureExtractor
from .mot import MOT
from .devmem import Frame, nv12_frame, pixel_frame
from .multicamera import MultiCameraMOT
from .multistream import MultiStreamMOT
from . import models
