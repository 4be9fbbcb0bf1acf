"""CPU: the NV12 -> BGR restatement (oracle/nv12.py) against cv2.cvtColor on every (Y, U, V) triple, and the NV12 frame
descriptor's parsing (fastmot_b200.devmem): the three accepted forms and the rejected ones."""
import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from oracle import nv12 as onv
from fastmot_b200 import devmem


def _all_triples_frame():
    """A 512 x 32768 NV12 frame holding every (Y, U, V) once: block row i has U = i, block columns 64 j .. 64 j + 63
    have V = j, and those 64 2x2 blocks carry Y = 0..255."""
    H, W = 2 * 256, 128 * 256
    blk = np.empty((2, 128), np.uint8)
    yv = np.arange(256, dtype=np.uint8).reshape(64, 4)
    blk[0, 0::2], blk[0, 1::2], blk[1, 0::2], blk[1, 1::2] = yv[:, 0], yv[:, 1], yv[:, 2], yv[:, 3]
    Y = np.tile(blk, (256, 256))
    UV = np.empty((H // 2, W // 2, 2), np.uint8)
    UV[..., 0] = np.arange(256, dtype=np.uint8)[:, None]
    UV[..., 1] = np.repeat(np.arange(256, dtype=np.uint8), 64)[None, :]
    return np.concatenate([Y, UV.reshape(H // 2, W)], 0)


def test_oracle_equals_cv2_on_all_yuv_triples():
    yuv = _all_triples_frame()
    # every triple is present
    h = yuv.shape[0] * 2 // 3
    uv = yuv[h:].reshape(h // 2, -1, 2)
    U = np.repeat(np.repeat(uv[..., 0], 2, 0), 2, 1).astype(np.int64)
    V = np.repeat(np.repeat(uv[..., 1], 2, 0), 2, 1).astype(np.int64)
    key = (yuv[:h].astype(np.int64) << 16) | (U << 8) | V
    assert np.unique(key).size == 1 << 24
    want = cv2.cvtColor(yuv, cv2.COLOR_YUV2BGR_NV12)
    got = onv.nv12_to_bgr(yuv)
    assert got.shape == want.shape and got.dtype == np.uint8
    assert int((got != want).sum()) == 0


def test_bgr_to_nv12_round_trip_layout():
    """bgr_to_nv12 is cv2's I420 with U and V interleaved: its NV12 and I420 decodes agree."""
    rng = np.random.default_rng(0)
    bgr = rng.integers(0, 256, (48, 64, 3), dtype=np.uint8)
    nv = onv.bgr_to_nv12(bgr)
    i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
    assert nv.shape == (72, 64)
    np.testing.assert_array_equal(cv2.cvtColor(nv, cv2.COLOR_YUV2BGR_NV12), cv2.cvtColor(i420, cv2.COLOR_YUV2BGR_I420))


# ---------------------------------------------------------------------------------------------------- descriptors
def test_descriptor_host_array():
    f = devmem.nv12_frame(np.zeros((1620, 1920), np.uint8))
    assert (f.format, f.size, f.on_device) == ("NV12", (1920, 1080), False)


def test_descriptor_pitched_tensor_layout():
    """A (3H/2, W) view with row stride W + 64 (CPU tensor: the layout check does not look at the device)."""
    surf = torch.zeros(1620, 1920 + 64, dtype=torch.uint8)
    f = devmem.nv12_layout(surf[:, :1920])
    assert (f.size, f.y_pitch, f.uv_pitch) == ((1920, 1080), 1984, 1984)
    assert f.uv.data_ptr() == surf.data_ptr() + 1080 * 1984
    with pytest.raises(ValueError, match="cuda"):
        devmem.nv12_frame(surf[:, :1920])


def test_descriptor_two_planes_layout():
    """A 1088-row decoder surface: Y = rows 0..1079, UV = rows 1088..1627, row stride 2048."""
    surf = torch.zeros(1088 + 544, 2048, dtype=torch.uint8)
    f = devmem.nv12_layout((surf[:1080, :1920], surf[1088:1088 + 540, :1920]))
    assert (f.size, f.y_pitch, f.uv_pitch) == ((1920, 1080), 2048, 2048)
    assert f.uv.data_ptr() == surf.data_ptr() + 1088 * 2048
    with pytest.raises(ValueError, match="cuda"):
        devmem.nv12_frame((surf[:1080, :1920], surf[1088:1088 + 540, :1920]))


@pytest.mark.parametrize("bad, what", [
    (np.zeros((1620, 1920), np.uint16), "uint8"),
    (np.zeros((1080, 1920, 3), np.uint8), r"\(3H/2, W\)"),
    (np.zeros((1621, 1920), np.uint8), r"\(3H/2, W\)"),
    (np.zeros((1620, 1919), np.uint8), "even"),
    (np.zeros((0, 1920), np.uint8), "even"),
    (torch.zeros(1620, 1920, dtype=torch.int16), "uint8"),
    (torch.zeros(1620, 1920, 2, dtype=torch.uint8), r"\(3H/2, W\)"),
    (torch.zeros(1620, 3840, dtype=torch.uint8)[:, ::2], "stride"),
    (torch.zeros(1620 * 1920, dtype=torch.uint8).as_strided((1620, 1920), (1900, 1)), "stride"),
    ((torch.zeros(1080, 1920, dtype=torch.uint8), torch.zeros(540, 1918, dtype=torch.uint8)), r"shape \(540, 1920\)"),
    ((torch.zeros(1080, 1920, dtype=torch.uint8), torch.zeros(541, 1920, dtype=torch.uint8)), r"shape \(540, 1920\)"),
    ((torch.zeros(1081, 1920, dtype=torch.uint8), torch.zeros(540, 1920, dtype=torch.uint8)), "even"),
    ((torch.zeros(1080, 1920, dtype=torch.uint8),), "pair"),
    ("frame.yuv", "ndarray or cuda tensor"),
])
def test_descriptor_rejects(bad, what):
    with pytest.raises(ValueError, match=what):
        devmem.nv12_layout(bad)
