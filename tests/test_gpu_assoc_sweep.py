"""GPU sweep of the fp64 Kalman and association kernels (csrc/kalman.cu, csrc/assoc.cu, csrc/assoc_lsa_block.cu,
csrc/assoc_cascade.cu) against the float64 restatements in oracle/kalman.py and oracle/assoc.py, at the flags,
shapes and thresholds the tracker uses and at the limits of each entry point.

Every kernel here computes a plain fp64 formula, so the bounds are tight: 1e-9 relative for values whose operation
order differs from numpy's (8x8 products, 4x4 solves, dot products), bit-exact where the order is the same (IoU,
occlusion, create, rounding, assignments).  Pools are filled with NaN-pattern sentinels so that a launch which reads
or writes a slot it was not given is caught.  Each test prints its worst error / tolerance ratio under `pytest -s`.
"""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CAP = 2048                  # MultiTracker's default pool_capacity
FRAME = (1920, 1080)
FRAME_RECT = [0, 0, FRAME[0] - 1, FRAME[1] - 1]
INF = 1e5                   # FM_INF_COST
CHI2 = 9.4877               # FM_CHI_SQ_INV_95
BOUNDARY_TOL = 1e-9


def _sentinel(shape, tag):
    """float64 NaNs with distinct payloads: a copy from a wrong slot changes the bits."""
    n = int(np.prod(shape))
    bits = np.int64(0x7FF4000000000000) + (np.int64(tag) << np.int64(36)) + np.arange(n, dtype=np.int64)
    return bits.view(np.float64).reshape(shape)


def _sentinel32(shape, tag):
    n = int(np.prod(shape))
    bits = np.int32(0x7F800001) + np.int32(tag << 21) + np.arange(n, dtype=np.int32)
    return bits.view(np.float32).reshape(shape)


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _report(name, **vals):
    print(f"[{name}] " + ", ".join(f"{k} {v:.3g}" if isinstance(v, float) else f"{k} {v}" for k, v in vals.items()))


# ------------------------------------------------------------------------------------------------------------------
# Kalman states
# ------------------------------------------------------------------------------------------------------------------
def _boxes(rng, n):
    """tlbr boxes with widths / heights below 50 px (0.08 * w < 4 and 0.14 * w < 5), above 50 px, of 1 px and wider
    than the frame, starting at negative coordinates as well."""
    x1 = rng.uniform(-300., 2000., n)
    y1 = rng.uniform(-200., 1100., n)

    def side(frame):
        kind = rng.integers(0, 4, n)
        return np.select([kind == 0, kind == 1, kind == 2],
                         [rng.uniform(2., 50., n), rng.uniform(50., 400., n), np.ones(n)],
                         rng.uniform(frame, 1.6 * frame, n))
    w, h = side(FRAME[0]), side(FRAME[1])
    return np.stack([x1, y1, x1 + w - 1., y1 + h - 1.], 1)


# exact boxes: x.5 means (round half to even) and integer boxes whose ios with the frame is exactly 0.5 or just below
_SPECIAL = np.array([[100.5, 200.5, 180.5, 260.5],
                     [101.5, -3.5, 151.5, 40.5],
                     [-50., 100., 49., 199.],       # ios 50/100 = 0.5: not lost
                     [-51., 100., 48., 199.],       # ios 0.49: lost
                     [1870., 500., 1969., 599.],    # ios 0.5 at the right edge
                     [300., 1030., 399., 1129.],    # ios 0.5 at the bottom edge
                     [7., 9., 7., 9.],              # 1 px
                     [-2.5, -0.5, 0.5, 2.5]])


def _random_h(rng, persp=2e-5):
    th = rng.normal(0, 0.01)
    s = 1. + rng.normal(0, 0.01)
    return np.array([[s * np.cos(th), -s * np.sin(th), rng.normal(0, 5)],
                     [s * np.sin(th), s * np.cos(th), rng.normal(0, 5)],
                     [rng.normal(0, persp), rng.normal(0, persp), 1.]])


def _homographies():
    th, s = 0.05, 1.03
    return {
        "identity": np.eye(3),
        "translation": np.array([[1., 0., 12.25], [0., 1., -7.5], [0., 0., 1.]]),
        "rotation_scale": np.array([[s * np.cos(th), -s * np.sin(th), 30.], [s * np.sin(th), s * np.cos(th), -20.],
                                    [0., 0., 1.]]),
        # strong perspective: a = g . p + 1 ranges over about [0.8, 1.5] on these boxes, the ia^3 term matters
        "perspective": np.array([[1.02, 0.01, 5.], [-0.015, 0.99, 3.], [1e-4, -0.8e-4, 1.]]),
    }


def _chain_states(rng, ko, n, steps=3):
    """States with non-diagonal covariances and velocities (create + a few warp / predict / flow-update rounds of
    the oracle); the boxes are then reset to the designed ones."""
    from oracle.kalman import FLOW
    tlbr = _boxes(rng, n)
    k = min(n, len(_SPECIAL))
    tlbr[:k] = _SPECIAL[:k]
    mean, cov = ko.create(tlbr)
    for _ in range(steps):
        mean, cov = ko.warp(mean, cov, _random_h(rng))
        mean, cov = ko.predict(mean, cov)
        mean, cov = ko.update(mean, cov, mean[:, :4] + rng.normal(0, 3, (n, 4)), FLOW, rng.uniform(1, 4, n))
    mean[:, :4] = tlbr
    return mean, cov


def _oracle_step(ko, mean, cov, flags, H, meas, has, mult):
    from fastmot_b200.kalman_filter import FM_KF_WARP, FM_KF_PREDICT, FM_KF_UPDATE, FM_KF_MEAS_DET
    from oracle.kalman import FLOW, DETECTOR
    if flags & FM_KF_WARP:
        mean, cov = ko.warp(mean, cov, H)
    if flags & FM_KF_PREDICT:
        mean, cov = ko.predict(mean, cov)
    if flags & FM_KF_UPDATE and has.any():
        mu, cu = ko.update(mean[has], cov[has], meas[has], DETECTOR if flags & FM_KF_MEAS_DET else FLOW, mult[has])
        mean, cov = mean.copy(), cov.copy()
        mean[has], cov[has] = mu, cu
    return mean, cov


class _KfPools:
    """mean / cov / tlbr pools of capacity CAP on the device, sentinels outside `slots`."""

    def __init__(self, slots, mean, cov, tag=1):
        self.slots = slots
        self.h_mean = _sentinel((CAP, 8), tag)
        self.h_cov = _sentinel((CAP, 64), tag + 1)
        self.h_tlbr = _sentinel((CAP, 4), tag + 2)
        self.h_mean[slots] = mean
        self.h_cov[slots] = cov.reshape(-1, 64)
        self.h_tlbr[slots] = 0.
        self.upload()

    def upload(self):
        from gpu_util import dev
        self.mean, self.cov, self.tlbr = dev(self.h_mean), dev(self.h_cov), dev(self.h_tlbr)

    def fetch(self):
        from gpu_util import host
        return host(self.mean), host(self.cov), host(self.tlbr)

    def untouched_ok(self, got):
        """every slot outside `slots` is bit-identical to its sentinel"""
        other = np.ones(CAP, bool)
        other[self.slots] = False
        return all(_same_bits(g[other], w[other]) for g, w in zip(got, (self.h_mean, self.h_cov, self.h_tlbr)))


def _check_state(got_mean, got_cov, want_mean, want_cov):
    """mean within 1e-9 (1 + |want|); cov within 1e-9 max |cov| of the track.  Returns the worst ratios."""
    rm = np.abs(got_mean - want_mean) / (1e-9 * (1. + np.abs(want_mean)))
    scale = np.abs(want_cov).reshape(len(want_cov), -1).max(1)
    rc = np.abs(got_cov - want_cov) / (1e-9 * scale[:, None, None])
    wm, wc = float(rm.max(initial=0.)), float(rc.max(initial=0.))
    assert np.all(np.isfinite(got_mean)) and np.all(np.isfinite(got_cov))
    assert wm <= 1. and wc <= 1., (wm, wc, np.unravel_index(np.argmax(rm), rm.shape))
    return wm, wc


def _check_round(got_mean, want_mean, out_tlbr, pool_tlbr, out_lost):
    """out_tlbr / tlbr_pool = rint(mean[:4]) and out_lost = ios(rint box, frame) < 0.5, exactly, on the kernel's own
    mean; and against the oracle's mean except where that lies within 1e-9 of x.5 and the two means differ.
    Returns the number of excluded coordinates."""
    from oracle.assoc import ios
    r = np.rint(got_mean[:, :4])
    assert np.array_equal(out_tlbr, r)
    assert np.array_equal(pool_tlbr, r)
    assert np.array_equal(out_lost, (ios(r, FRAME_RECT) < 0.5).astype(np.uint8))
    w = want_mean[:, :4]
    rw = np.rint(w)
    near = (np.abs(w - (np.floor(w) + 0.5)) <= BOUNDARY_TOL * (1. + np.abs(w))) & (got_mean[:, :4] != w)
    assert np.array_equal(r[~near], rw[~near])
    keep = ~near.any(1)
    assert np.array_equal(out_lost[keep], (ios(rw, FRAME_RECT) < 0.5).astype(np.uint8)[keep])
    return int(near.sum())


# ------------------------------------------------------------------------------------------------------------------
# 1. fm_kalman_create_batched / fm_kalman_step_batched
# ------------------------------------------------------------------------------------------------------------------
KF_SIZES = [1, 63, 64, 65, 200, 2048]


@pytest.mark.parametrize("n", KF_SIZES)
def test_kalman_create_batched_bit_exact(lib, n):
    """create with a tlbr_idx indirection (permuted, repeated) into scattered slots == KalmanOracle.create bit for
    bit; tlbr_pool gets the box; every other slot keeps its sentinel."""
    from gpu_util import dev, kalman_params
    from fastmot_b200.devmem import ptr
    from oracle.kalman import KalmanOracle
    kf, ko = kalman_params(), KalmanOracle(1 / 30)
    rng = np.random.default_rng(10 + n)
    slots = rng.permutation(CAP)[:n].astype(np.int32)
    tlbr = _boxes(rng, n + 5)
    tlbr[:len(_SPECIAL)] = _SPECIAL[:min(len(_SPECIAL), n + 5)]
    idx = rng.integers(0, n + 5, n).astype(np.int32)
    P = _KfPools(slots, np.zeros((n, 8)), np.zeros((n, 8, 8)))
    P.h_tlbr[slots] = _sentinel((n, 4), 9)      # create must overwrite these
    P.upload()
    d_slots, d_tlbr, d_idx = dev(slots), dev(tlbr), dev(idx)
    kf.create_batched(P.mean, P.cov, P.tlbr, ptr(d_slots), ptr(d_tlbr), ptr(d_idx), n)
    got = P.fetch()
    want_m, want_c = ko.create(tlbr[idx])
    assert _same_bits(got[0][slots], want_m)
    assert _same_bits(got[1][slots], want_c.reshape(n, 64))
    assert _same_bits(got[2][slots], tlbr[idx])
    assert P.untouched_ok(got)


@pytest.mark.parametrize("n", KF_SIZES)
def test_kalman_step_every_flag_combination(lib, n):
    """All 32 combinations of WARP / PREDICT / UPDATE / MEAS_DET / MEAS_BY_SLOT on scattered slots, cycling through
    four homographies, has_meas NULL / per item / by slot, and the noise multiplier NULL / mult_num /
    mult_num / mult_den_pool[slot]; each launch starts from the same state and is compared to the oracle."""
    from gpu_util import dev, host, kalman_params
    from fastmot_b200.devmem import ptr
    from fastmot_b200.kalman_filter import FM_KF_WARP, FM_KF_PREDICT, FM_KF_UPDATE, FM_KF_MEAS_BY_SLOT
    from oracle.kalman import KalmanOracle
    kf, ko = kalman_params(), KalmanOracle(1 / 30)
    rng = np.random.default_rng(100 + n)
    slots = rng.permutation(CAP)[:n].astype(np.int32)
    mean0, cov0 = _chain_states(rng, ko, n)
    P = _KfPools(slots, mean0, cov0)
    Hs = _homographies()
    names = list(Hs)
    meas_item = mean0[:, :4] + rng.normal(0, 4, (n, 4))
    meas_pool = _sentinel((CAP, 4), 5)
    meas_pool[slots] = meas_item
    has_item = rng.random(n) < 0.7
    has_pool = rng.random(CAP) < 0.5
    has_pool[slots] = has_item
    num = rng.integers(1, 30, n).astype(np.float64)
    den_pool = rng.uniform(0.2, 1.0, CAP)
    d_slots = dev(slots)
    d_meas = {False: dev(meas_item), True: dev(meas_pool)}
    d_has = {False: dev(has_item.astype(np.uint8)), True: dev(has_pool.astype(np.uint8))}
    d_num, d_den_ = dev(num), dev(den_pool)
    worst_m = worst_c = 0.
    excluded = 0
    for f in range(32):
        hname = names[(f // 2 + n) % 4]
        hm_mode, mu_mode = f % 3, f % 5
        by_slot = bool(f & FM_KF_MEAS_BY_SLOT)
        P.upload()
        d_H = dev(Hs[hname].reshape(9))
        out = dev(_sentinel((n, 4), 7))
        lost = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
        kf.step_batched(P.mean, P.cov, P.tlbr, ptr(d_slots), n, f, homography=ptr(d_H),
                        meas=ptr(d_meas[by_slot]), has_meas=None if hm_mode == 0 else ptr(d_has[by_slot]),
                        mult_num=None if mu_mode == 0 else ptr(d_num),
                        mult_den_pool=ptr(d_den_) if mu_mode >= 2 else None,
                        frame_size=FRAME, out_tlbr=ptr(out), out_lost=ptr(lost))
        got = P.fetch()
        assert P.untouched_ok(got), f
        has = np.ones(n, bool) if hm_mode == 0 else has_item
        mult = np.ones(n) if mu_mode == 0 else (num / 1.0 if mu_mode == 1 else num / den_pool[slots])
        wm, wc = _oracle_step(ko, mean0, cov0, f, Hs[hname], meas_item, has, mult)
        gm, gc = got[0][slots], got[1][slots].reshape(n, 8, 8)
        if not f & (FM_KF_WARP | FM_KF_PREDICT) and not (f & FM_KF_UPDATE and has.any()):
            assert _same_bits(gm, mean0) and _same_bits(gc, cov0.reshape(n, 8, 8)), f
        if f & FM_KF_WARP and hname == "identity" and not f & (FM_KF_PREDICT | FM_KF_UPDATE):
            assert np.array_equal(gm, mean0) and np.array_equal(gc, cov0), f
        rm, rc = _check_state(gm, gc, wm, wc)
        worst_m, worst_c = max(worst_m, rm), max(worst_c, rc)
        excluded += _check_round(gm, wm, host(out), got[2][slots], host(lost))
    assert excluded <= 4, excluded
    _report(f"kalman flags n={n}", mean_err_over_tol=worst_m, cov_err_over_tol=worst_c, excluded=excluded)


def test_kalman_h_ok_and_hold_are_no_ops(lib):
    """*h_ok == 0 or *hold != 0: the launch writes nothing, in the pools or in out_tlbr / out_lost; h_ok = 1 with
    hold = 0 runs the step."""
    from gpu_util import dev, host, kalman_params
    from fastmot_b200.devmem import ptr
    from fastmot_b200.kalman_filter import FM_KF_WARP, FM_KF_PREDICT, FM_KF_UPDATE, FM_KF_MEAS_BY_SLOT
    from oracle.kalman import KalmanOracle
    kf, ko = kalman_params(), KalmanOracle(1 / 30)
    rng = np.random.default_rng(7)
    n = 200
    slots = rng.permutation(CAP)[:n].astype(np.int32)
    mean0, cov0 = _chain_states(rng, ko, n)
    P = _KfPools(slots, mean0, cov0)
    H = _homographies()["perspective"]
    meas_pool = _sentinel((CAP, 4), 5)
    meas_pool[slots] = mean0[:, :4] + rng.normal(0, 4, (n, 4))
    has_pool = np.ones(CAP, np.uint8)
    num = rng.integers(1, 30, n).astype(np.float64)
    den_pool = rng.uniform(0.2, 1.0, CAP)
    d = {k: dev(v) for k, v in dict(slots=slots, H=H.reshape(9), meas=meas_pool, has=has_pool, num=num,
                                    den=den_pool, zero=np.zeros(1, np.int32), one=np.ones(1, np.int32)).items()}
    flags = FM_KF_WARP | FM_KF_PREDICT | FM_KF_UPDATE | FM_KF_MEAS_BY_SLOT
    out_s = _sentinel((n, 4), 7)

    def run(h_ok, hold):
        P.upload()
        out = dev(out_s)
        lost = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
        kf.step_batched(P.mean, P.cov, P.tlbr, ptr(d["slots"]), n, flags, homography=ptr(d["H"]),
                        h_ok=None if h_ok is None else ptr(d["one" if h_ok else "zero"]),
                        hold=None if hold is None else ptr(d["one" if hold else "zero"]),
                        meas=ptr(d["meas"]), has_meas=ptr(d["has"]), mult_num=ptr(d["num"]),
                        mult_den_pool=ptr(d["den"]), frame_size=FRAME, out_tlbr=ptr(out), out_lost=ptr(lost))
        return P.fetch(), host(out), host(lost)

    for h_ok, hold in ((0, None), (0, 0), (0, 1), (1, 1), (None, 1)):
        got, out, lost = run(h_ok, hold)
        assert all(_same_bits(g, w) for g, w in zip(got, (P.h_mean, P.h_cov, P.h_tlbr))), (h_ok, hold)
        assert _same_bits(out, out_s) and np.all(lost == 7), (h_ok, hold)
    for h_ok, hold in ((1, 0), (1, None), (None, 0)):
        got, out, lost = run(h_ok, hold)
        wm, wc = _oracle_step(ko, mean0, cov0, flags, H, meas_pool[slots], np.ones(n, bool), num / den_pool[slots])
        rm, rc = _check_state(got[0][slots], got[1][slots].reshape(n, 8, 8), wm, wc)
        _check_round(got[0][slots], wm, out, got[2][slots], lost)
        assert P.untouched_ok(got)
    _report("kalman h_ok/hold", mean_err_over_tol=rm, cov_err_over_tol=rc)


def test_kalman_tracker_chain_30_frames(lib):
    """The tracker's pattern for 30 frames on 200 scattered tracks, never re-synchronised with the oracle:
    every frame WARP|PREDICT|UPDATE|MEAS_BY_SLOT with a fresh H, klt_ok = 0 for some tracks, mult_num = max(2 age, 1)
    over the inlier-ratio pool; every 5th frame UPDATE|MEAS_DET of a subset with per-item detections."""
    from gpu_util import dev, host, kalman_params
    from fastmot_b200.devmem import ptr
    from fastmot_b200.kalman_filter import (FM_KF_WARP, FM_KF_PREDICT, FM_KF_UPDATE, FM_KF_MEAS_BY_SLOT,
                                            FM_KF_MEAS_DET)
    from oracle.kalman import KalmanOracle
    kf, ko = kalman_params(), KalmanOracle(1 / 30)
    rng = np.random.default_rng(30)
    n = 200
    slots = rng.permutation(CAP)[:n].astype(np.int32)
    tlbr = _boxes(rng, n)
    P = _KfPools(slots, np.zeros((n, 8)), np.zeros((n, 8, 8)))
    d_slots, d_tlbr = dev(slots), dev(tlbr)
    kf.create_batched(P.mean, P.cov, P.tlbr, ptr(d_slots), ptr(d_tlbr), None, n)
    mean, cov = ko.create(tlbr)
    got = P.fetch()
    assert _same_bits(got[0][slots], mean) and _same_bits(got[1][slots], cov.reshape(n, 64))
    h_ok = dev(np.ones(1, np.int32))
    age = rng.integers(0, 5, n)
    worst_m = worst_c = 0.
    excluded = 0
    for frame in range(30):
        H = _random_h(rng, persp=2e-5)
        meas_pool = _sentinel((CAP, 4), 3)
        meas_pool[slots] = mean[:, :4] + rng.normal(0, 3, (n, 4))
        klt_ok = np.zeros(CAP, np.uint8)
        klt_ok[slots] = rng.random(n) > 0.2
        ratio_pool = rng.uniform(0.3, 1.0, CAP)
        num = np.maximum(2. * age, 1.)
        d = [dev(x) for x in (H.reshape(9), meas_pool, klt_ok, num, ratio_pool)]
        out = dev(_sentinel((n, 4), 7))
        lost = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
        kf.step_batched(P.mean, P.cov, P.tlbr, ptr(d_slots), n,
                        FM_KF_WARP | FM_KF_PREDICT | FM_KF_UPDATE | FM_KF_MEAS_BY_SLOT, homography=ptr(d[0]),
                        h_ok=ptr(h_ok), meas=ptr(d[1]), has_meas=ptr(d[2]), mult_num=ptr(d[3]),
                        mult_den_pool=ptr(d[4]), frame_size=FRAME, out_tlbr=ptr(out), out_lost=ptr(lost))
        mean, cov = _oracle_step(ko, mean, cov, FM_KF_WARP | FM_KF_PREDICT | FM_KF_UPDATE, H, meas_pool[slots],
                                 klt_ok[slots].astype(bool), num / ratio_pool[slots])
        got = P.fetch()
        rm, rc = _check_state(got[0][slots], got[1][slots].reshape(n, 8, 8), mean, cov)
        worst_m, worst_c = max(worst_m, rm), max(worst_c, rc)
        excluded += _check_round(got[0][slots], mean, host(out), got[2][slots], host(lost))
        age += 1
        if frame % 5 == 4:
            sub = np.sort(rng.permutation(n)[:int(0.7 * n)])
            ns = len(sub)
            z = np.rint(mean[sub, :4] + rng.normal(0, 2, (ns, 4)))
            d2 = [dev(slots[sub]), dev(z)]
            out = dev(_sentinel((ns, 4), 8))
            lost = torch.full((ns,), 7, dtype=torch.uint8, device="cuda")
            kf.step_batched(P.mean, P.cov, P.tlbr, ptr(d2[0]), ns, FM_KF_UPDATE | FM_KF_MEAS_DET, meas=ptr(d2[1]),
                            frame_size=FRAME, out_tlbr=ptr(out), out_lost=ptr(lost))
            mean, cov = mean.copy(), cov.copy()
            mean[sub], cov[sub] = _oracle_step(ko, mean[sub], cov[sub], FM_KF_UPDATE | FM_KF_MEAS_DET, None, z,
                                               np.ones(ns, bool), np.ones(ns))
            got = P.fetch()
            rm, rc = _check_state(got[0][slots], got[1][slots].reshape(n, 8, 8), mean, cov)
            worst_m, worst_c = max(worst_m, rm), max(worst_c, rc)
            excluded += _check_round(got[0][slots[sub]], mean[sub], host(out), got[2][slots[sub]], host(lost))
            age[sub] = 0
    assert P.untouched_ok(P.fetch())
    assert excluded <= 4, excluded
    _report("kalman 30-frame chain", mean_err_over_tol=worst_m, cov_err_over_tol=worst_c, excluded=excluded)


# ------------------------------------------------------------------------------------------------------------------
# 2. fm_motion_distance and fm_matching_cost
# ------------------------------------------------------------------------------------------------------------------
MC_CAP = 512
MC_SHAPES = [(1, 1), (1, 9), (1, 200), (1, 300), (200, 1), (200, 9), (200, 200), (200, 300)]


@pytest.fixture(scope="module")
def tracks200():
    from oracle.kalman import KalmanOracle
    rng = np.random.default_rng(200)
    ko = KalmanOracle(1 / 30)
    mean, cov = _chain_states(rng, ko, 200)
    return mean, cov


def _projected(mean, cov):
    from oracle.kalman import KalmanOracle, DETECTOR
    pm, S = KalmanOracle(1 / 30).project(mean, cov, DETECTOR)
    return pm, np.linalg.cholesky(S)


def _dets_around(rng, mean, cov, n_rows):
    """Detections around random tracks at Mahalanobis distances from well inside to well outside the gate."""
    pm, L = _projected(mean, cov)
    home = rng.integers(0, len(mean), n_rows)
    y = rng.normal(size=(n_rows, 4)) * rng.choice([0.3, 1.2, 3.0], n_rows)[:, None]
    return pm[home] + np.einsum('nij,nj->ni', L[home], y)


def _at_gate(mean, cov, t, factor):
    """A detection at squared Mahalanobis distance CHI2 * factor from track t."""
    pm, L = _projected(mean[t:t + 1], cov[t:t + 1])
    y = np.array([0.5, -0.5, 0.5, 0.5]) * np.sqrt(CHI2 * factor)
    return pm[0] + L[0] @ y


@pytest.mark.parametrize("nt,nd", MC_SHAPES)
@pytest.mark.parametrize("use_slots", [False, True])
def test_motion_distance(lib, tracks200, nt, nd, use_slots):
    from gpu_util import dev, host, kalman_params
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    from oracle.kalman import KalmanOracle
    kf, ko = kalman_params(), KalmanOracle(1 / 30)
    rng = np.random.default_rng(nt * 1000 + nd + use_slots)
    mean, cov = tracks200[0][:nt], tracks200[1][:nt]
    slots = rng.permutation(MC_CAP)[:nt].astype(np.int32) if use_slots else np.arange(nt, dtype=np.int32)
    pm, pc = _sentinel((MC_CAP, 8), 1), _sentinel((MC_CAP, 64), 2)
    pm[slots], pc[slots] = mean, cov.reshape(nt, 64)
    z = _dets_around(rng, mean, cov, nd)
    z[0] = _at_gate(mean, cov, 0, 1.0)
    out = torch.full((nt, nd), -1., dtype=torch.float64, device="cuda")
    d = [dev(x) for x in (pm, pc, slots, z)]
    _lib.check(lib.fm_motion_distance(ptr(d[0]), ptr(d[1]), ptr(d[2]) if use_slots else None, nt, ptr(d[3]), nd,
                                      kf.params, ptr(out), stream_ptr()), "fm_motion_distance")
    got = host(out)
    want = ko.motion_distance(mean, cov, z)
    r = float((np.abs(got - want) / (1e-9 * (1. + np.abs(want)))).max())
    assert r <= 1., r
    _report(f"motion_distance {nt}x{nd} slots={use_slots}", err_over_tol=r)


def _cdist(XA, XB, metric, empty, fill):
    from oracle import assoc
    step = max(1, (1 << 24) // max(1, XB.shape[0] * XB.shape[1])) if metric == "euclidean" else len(XA)
    return np.concatenate([assoc.cdist(XA[i:i + step], XB, metric, empty[i:i + step], fill)
                           for i in range(0, len(XA), step)], 0)


def _sparse_pattern(rng, dim):
    """A feature whose cosine with itself is exactly 0 in any summation order: 16 entries of +-0.25 (norm 1)."""
    p = np.zeros(dim, np.float32)
    if dim < 16:
        p[0] = 1.
        return p
    p[rng.permutation(dim)[:16]] = rng.choice([-0.25, 0.25], 16)
    return p


def _matching_case(lib, mean, cov, rng, nt, nd, dim, metric, mw, max_cost, use_slots, valid_mode, use_occ,
                   sel_mode, fill, labels_mode):
    """One fm_matching_cost launch against cdist -> fuse_motion -> gate_cost of the oracle.  Returns the worst
    error / tolerance and the number of entries excluded as lying within 1e-9 of a gate."""
    from gpu_util import Keep, dev, host, kalman_params
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    from oracle import assoc
    from oracle.kalman import KalmanOracle
    kf, ko = kalman_params(), KalmanOracle(1 / 30)
    K = Keep()
    mean, cov = mean[:nt], cov[:nt]
    slots = rng.permutation(MC_CAP)[:nt].astype(np.int32) if use_slots else np.arange(nt, dtype=np.int32)
    n_rows = nd if sel_mode == 0 else nd + 13
    if sel_mode == 0:
        sel = np.arange(nd, dtype=np.int32)
    else:
        sel = rng.permutation(n_rows)[:nd].astype(np.int32)
        if sel_mode == 2 and nd > 8:          # repeated indices at the end
            sel[-(nd // 4):] = rng.choice(sel[:nd - nd // 4], nd // 4)
    feat = rng.normal(size=(MC_CAP, dim)).astype(np.float32)
    feat /= np.linalg.norm(feat, axis=1, keepdims=True)
    emb = rng.normal(size=(n_rows, dim)).astype(np.float32)
    emb /= np.linalg.norm(emb, axis=1, keepdims=True)
    det = _dets_around(rng, mean, cov, n_rows)
    valid = np.ones(MC_CAP, np.uint8) if valid_mode == 0 else (rng.random(MC_CAP) > 0.2).astype(np.uint8)
    occ = (rng.random(n_rows) < 0.15).astype(np.uint8)
    tl = rng.integers(0, 2, nt).astype(np.int64)
    dl = rng.integers(0, 2, n_rows).astype(np.int64)
    # column 0: an exact pair with track 0 (identical features, box at the track's mean: cost exactly 0)
    # columns 1-3: Mahalanobis distance to track 0 just inside, at and just outside the gate; columns 4, 5: exact
    # pairs with tracks 1 and 2.  The first nd - nd // 4 entries of det_sel are distinct.
    pattern = {}
    for j, t in ((0, 0), (4, 1 % nt), (5, 2 % nt)):
        if j < nd:
            if t not in pattern:
                pattern[t] = _sparse_pattern(rng, dim)
                feat[slots[t]] = pattern[t]
            emb[sel[j]] = pattern[t]
            det[sel[j]] = mean[t, :4]
            dl[sel[j]] = tl[t]
            valid[slots[t]] = 1
            occ[sel[j]] = 0
    for j, fac in ((1, 1 - 1e-7), (2, 1.), (3, 1 + 1e-7)):
        if j < nd:
            det[sel[j]] = _at_gate(mean, cov, 0, fac)
    pm, pc = _sentinel((MC_CAP, 8), 1), _sentinel((MC_CAP, 64), 2)
    pm[slots], pc[slots] = mean, cov.reshape(nt, 64)
    out = torch.full((nt, nd), -1., dtype=torch.float64, device="cuda")
    rc = lib.fm_matching_cost(K(feat), None if valid_mode == 0 else K(valid), K(pm), K(pc),
                              K(slots) if use_slots else K(np.arange(nt, dtype=np.int32)),
                              K(tl) if labels_mode in (0, 2) else None, nt, K(emb), K(det),
                              K(dl) if labels_mode in (0, 1) else None, K(occ) if use_occ else None,
                              None if sel_mode == 0 else K(sel), nd, dim, 1 if metric == "cosine" else 0, fill, mw,
                              max_cost, kf.params, ptr(out), stream_ptr())
    _lib.check(rc, "fm_matching_cost")
    got = host(out)
    # reference
    empty = (valid[slots] == 0)[:, None] | ((occ[sel] != 0)[None, :] if use_occ else np.zeros((1, nd), bool))
    c = _cdist(feat[slots].astype(np.float64), emb[sel].astype(np.float64), metric, empty, fill)
    amb = np.zeros((nt, nd), bool)
    if mw >= 0:
        md = ko.motion_distance(mean, cov, det[sel])
        c = assoc.fuse_motion(c, md, mw)
        amb |= (np.abs(md - CHI2) <= BOUNDARY_TOL * CHI2) & (md != CHI2)
    if max_cost >= 0:
        amb |= (np.abs(c - max_cost) <= BOUNDARY_TOL) & (c != max_cost)
    gate_labels = labels_mode == 0
    want = assoc.gate_cost(c, tl if gate_labels else np.zeros(nt), dl[sel] if gate_labels else np.zeros(nd),
                           max_cost if max_cost >= 0 else None)
    assert amb.sum() <= 3, amb.sum()     # the at-gate detection, and rarely another
    assert np.array_equal((got == INF)[~amb], (want == INF)[~amb])
    fin = ~amb & (want != INF)
    r = np.abs(got - want)[fin] / (1e-9 * np.maximum(1., np.abs(want[fin])))
    worst = float(r.max(initial=0.))
    assert worst <= 1., worst
    if max_cost == 0.:
        assert got[0, 0] == 0.          # the exact pair sits exactly at the gate and passes it
    return worst, int(amb.sum())


@pytest.mark.parametrize("dim", [1, 31, 33, 128, 512, 2048, 8192])
@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_matching_cost_sweep(lib, tracks200, dim, metric):
    """Every (n_trk, n_det) of MC_SHAPES at this dim / metric; motion_weight, max_cost (off, the tracker's 0.9, and
    0 hit exactly by identical features), slots, feat_valid_pool, det_occluded, det_sel (identity, permuted,
    permuted with repeats), fill_val and the label arrays (both, trk NULL, det NULL, none) cycle across cases."""
    worst, excl = 0., 0
    for k, (nt, nd) in enumerate(MC_SHAPES):
        c = k + 8 * (dim % 7) + (metric == "cosine")
        rng = np.random.default_rng(c * 31 + dim)
        w, e = _matching_case(lib, *tracks200, rng, nt, nd, dim, metric,
                              mw=[-1., 0., 0.2, 1.][c % 4], max_cost=[-1., 0.9, 0.][c % 3],
                              use_slots=bool((c // 3) % 2), valid_mode=(c // 5) % 2, use_occ=bool((c // 7) % 2 == 0),
                              sel_mode=(c // 2) % 3, fill=[1.0, 0.35][(c // 11) % 2], labels_mode=(c // 4) % 4)
        worst, excl = max(worst, w), excl + e
    _report(f"matching_cost dim={dim} {metric}", err_over_tol=worst, excluded=excl)


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
@pytest.mark.parametrize("labels_mode", [0, 1, 2, 3])
@pytest.mark.parametrize("max_cost", [-1., 0.9, 0.])
def test_matching_cost_flag_grid(lib, tracks200, metric, labels_mode, max_cost):
    """Every motion_weight x label-array x max_cost combination at 200 x 200, dim 512."""
    worst, excl = 0., 0
    for mw in (-1., 0., 0.2, 1.):
        rng = np.random.default_rng(int(1000 * (mw + 1)) + 17 * labels_mode + 3)
        w, e = _matching_case(lib, *tracks200, rng, 200, 200, 512, metric, mw=mw, max_cost=max_cost, use_slots=True,
                              valid_mode=1, use_occ=True, sel_mode=2, fill=1.0, labels_mode=labels_mode)
        worst, excl = max(worst, w), excl + e
    _report(f"matching_cost grid {metric} labels={labels_mode} max={max_cost}", err_over_tol=worst, excluded=excl)


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
def test_matching_cost_tracker_calls(lib, tracks200, metric):
    """The two calls MultiTracker makes, with its arguments: appearance + motion (feat_valid_pool, labels,
    fm_find_occluded flags, fill = min(0.9 + 0.1, 1), motion_weight 0.2, max_cost 0.9, det_sel per stage or NULL
    in the fused cascade) and re-identification (no valid pool, no occlusion, fill 1, motion and gate off)."""
    worst, excl = 0., 0
    for k, (sel_mode, kw) in enumerate([
            (2, dict(mw=0.2, max_cost=0.9, valid_mode=1, use_occ=True, fill=min(0.9 + 0.1, 1.))),
            (0, dict(mw=0.2, max_cost=0.9, valid_mode=1, use_occ=True, fill=min(0.9 + 0.1, 1.))),
            (0, dict(mw=-1., max_cost=-1., valid_mode=0, use_occ=False, fill=1.0))]):
        rng = np.random.default_rng(50 + k)
        w, e = _matching_case(lib, *tracks200, rng, 200, 200, 512, metric, use_slots=True, sel_mode=sel_mode,
                              labels_mode=0, **kw)
        worst, excl = max(worst, w), excl + e
    _report(f"matching_cost tracker calls {metric}", err_over_tol=worst, excluded=excl)


# ------------------------------------------------------------------------------------------------------------------
# 3. fm_iou_cost and fm_find_occluded
# ------------------------------------------------------------------------------------------------------------------
def _int_boxes(rng, n, span=240):
    """Integer tlbr boxes in a small area (many overlaps), with zero and negative widths / heights."""
    x1 = rng.integers(-20, span, n)
    y1 = rng.integers(-20, span, n)
    w = rng.integers(-3, 60, n)
    h = rng.integers(-3, 60, n)
    return np.stack([x1, y1, x1 + w - 1, y1 + h - 1], 1).astype(np.float64)


@pytest.mark.parametrize("labels", ["both", "trk_null", "det_null"])
@pytest.mark.parametrize("max_cost", [1. - 0.4, -1.])
def test_iou_cost_bit_exact(lib, labels, max_cost):
    """300 tracks from scattered pool slots x 250 selected detections (75 000 > 65 536 entries, 293 CTAs) with
    permuted and repeated det_sel, labels and the tracker's gate 1 - iou_thresh; touching boxes (iw == 0), identical
    boxes, empty boxes and IoU exactly 0.4.  Bit-identical to iou_dist + gate_cost."""
    from gpu_util import Keep, host
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    from oracle import assoc
    rng = np.random.default_rng(3)
    nt, n_rows, nd = 300, 280, 250
    trk = _int_boxes(rng, nt)
    det = _int_boxes(rng, n_rows)
    near = rng.permutation(n_rows)[:n_rows // 2]         # half the detections are shifted copies of tracks
    det[near] = trk[rng.integers(0, nt, len(near))] + rng.integers(-3, 4, (len(near), 4))
    sel = rng.permutation(n_rows)[:nd].astype(np.int32)
    sel[-40:] = rng.choice(sel[:nd - 40], 40)
    trk[0] = [10, 10, 19, 19]
    det[sel[0]] = [12, 12, 19, 16]              # 8 x 5 inside a 10 x 10: IoU exactly 0.4, cost exactly 0.6
    det[sel[1]] = [20, 10, 29, 19]              # touches trk 0: iw == 0
    det[sel[2]] = trk[0]                        # identical
    trk[1] = [40, 40, 39, 60]                   # zero width
    trk[2] = [70, 70, 60, 60]                   # negative width and height
    tl = rng.integers(0, 3, nt).astype(np.int64)
    dl = rng.integers(0, 3, n_rows).astype(np.int64)
    tl[0] = dl[sel[0]] = dl[sel[1]] = dl[sel[2]] = 1
    slots = rng.permutation(CAP)[:nt].astype(np.int32)
    pool = _sentinel((CAP, 4), 4)
    pool[slots] = trk
    K = Keep()
    out = torch.full((nt, nd), -1., dtype=torch.float64, device="cuda")
    _lib.check(lib.fm_iou_cost(K(pool), K(slots), K(tl) if labels != "trk_null" else None, nt, K(det),
                               K(dl) if labels != "det_null" else None, K(sel), nd, max_cost, ptr(out),
                               stream_ptr()), "fm_iou_cost")
    got = host(out)
    c = assoc.iou_dist(trk, det[sel])
    gate = labels == "both"
    want = assoc.gate_cost(c, tl if gate else np.zeros(nt), dl[sel] if gate else np.zeros(nd),
                           max_cost if max_cost >= 0 else None)
    assert _same_bits(got, want)
    assert c[0, 0] == 0.6 and got[0, 0] == 0.6 and c[0, 1] == 1. and c[0, 2] == 0.
    n_pass = int((want < INF).sum()) if max_cost >= 0 else int((c < 1).sum())
    assert n_pass > 50
    _report(f"iou_cost labels={labels} max={max_cost}", bit_exact=True, finite=n_pass)


@pytest.mark.parametrize("n", [1, 127, 128, 129, 1000])
def test_find_occluded_bit_exact(lib, n):
    """Random integer boxes plus, far from them, a 10 x 10 box with exactly 70 of its 100 pixels covered (0.7 >=
    occlusion_thresh: occluded) and a 4 x 25 box with exactly 69 covered (not occluded)."""
    from gpu_util import Keep, host
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    from oracle import assoc
    rng = np.random.default_rng(n)
    boxes = _int_boxes(rng, n)
    special = np.array([[10000, 0, 10009, 9], [10000, 3, 10009, 9],          # 10 x 7 = 70 of 100
                        [20000, 0, 20003, 24], [20000, 2, 20002, 24]], float)  # 3 x 23 = 69 of 100
    if n >= 4:
        pos = rng.permutation(n)[:4]
        boxes[pos] = special
    out = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
    K = Keep()
    _lib.check(lib.fm_find_occluded(K(boxes), n, 0.7, ptr(out), stream_ptr()), "fm_find_occluded")
    got = host(out)
    want = assoc.find_occluded(boxes, 0.7)
    assert np.array_equal(got, want.astype(np.uint8))
    if n >= 4:
        assert want[pos[0]] and not want[pos[2]]
    _report(f"find_occluded n={n}", bit_exact=True, occluded=int(want.sum()))


# ------------------------------------------------------------------------------------------------------------------
# 4. fm_greedy_match, fm_lsa and fm_assoc_cascade at their limits
# ------------------------------------------------------------------------------------------------------------------
def _greedy_costs(rng, nr, nc, kind):
    if kind == "continuous":
        return rng.uniform(0, 1, (nr, nc))
    if kind == "quantised":
        return np.round(rng.uniform(0, 1, (nr, nc)) * 8) / 8
    return np.where(rng.random((nr, nc)) < 0.4, INF, rng.uniform(0, 1, (nr, nc)))


@pytest.mark.parametrize("shape", [(1, 1), (1, 300), (300, 1), (512, 512), (4096, 8), (8, 4096)])
@pytest.mark.parametrize("kind", ["continuous", "quantised", "inf"])
def test_greedy_match_vs_oracle(lib, shape, kind):
    """Matches in discovery order and the leftovers == oracle.assoc.greedy_match, with max_cost equal to one of the
    entries the scan reaches (`<=` matches it), the re-id threshold 0.45, and FM_INF_COST itself."""
    from gpu_util import run_greedy
    from fastmot_b200.tracker import MultiTracker
    from oracle import assoc
    nr, nc = shape
    rng = np.random.default_rng(nr * 7 + nc + len(kind))
    C = _greedy_costs(rng, nr, nc, kind)
    rows, cols = list(range(nr)), list(range(100, 100 + nc))
    full, _, _ = assoc.greedy_match(C, rows, cols, np.inf)
    hit = C[full[len(full) // 2][0], full[len(full) // 2][1] - 100]     # a cost the scan takes as its minimum
    n_match = 0
    for max_cost in sorted({hit, 0.45, INF}):
        c4r, order = run_greedy(C, max_cost)
        got = MultiTracker._split_greedy(c4r, order, nr, nc, rows, cols)
        want = assoc.greedy_match(C, rows, cols, max_cost)
        assert got[0] == want[0] and got[1] == want[1] and got[2] == want[2], (max_cost, len(got[0]), len(want[0]))
        n_match += len(want[0])
    c4r, _ = run_greedy(C, hit)
    assert any(C[r, c] == hit for r, c in enumerate(c4r) if c >= 0)      # the entry at max_cost was matched
    _report(f"greedy {shape} {kind}", bit_exact=True, matches=n_match)


def _lsa_want(C, rows, cols):
    want = np.full(C.shape[0], -1, np.int64)
    want[rows] = cols
    dem = (want >= 0) & (C[np.arange(len(want)), np.maximum(want, 0)] >= INF)
    return np.where(dem, -2 - want, want), int(dem.sum())


@pytest.mark.parametrize("shape", [(1200, 1300), (1300, 1200), (2048, 700), (1606, 40), (1607, 40), (40, 1607)])
def test_lsa_workspace_path_vs_scipy(lib, shape):
    """Shapes whose solver state exceeds 46 KB of shared memory run from the caller's global workspace; (1606, 40)
    is the largest of its family that still fits.  Continuous costs have a unique optimum, so the assignment must
    equal SciPy's; rows / columns of costs >= FM_INF_COST force demotions (-2 - c), also on the transposed side."""
    from scipy.optimize import linear_sum_assignment
    from gpu_util import run_lsa
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import stream_ptr
    nr, nc = shape
    rng = np.random.default_rng(nr + 3 * nc)
    C = rng.uniform(0, 1, (nr, nc))
    if nr <= nc:
        C[rng.permutation(nr)[:3]] = INF + rng.uniform(0, 1, (3, nc))     # these rows must take an INF column
    else:
        C[:, rng.permutation(nc)[:3]] = INF + rng.uniform(0, 1, (nr, 3))  # these columns must take an INF row
    smem = int(lib.fm_lsa_workspace_bytes(nr, nc)) <= 46 * 1024
    assert smem == (shape == (1606, 40))
    if not smem:      # without a workspace the call is refused, so this shape does run the workspace path
        assert lib.fm_lsa(None, nr, nc, None, None, None, stream_ptr()) != 0
    c4r, st = run_lsa(C)
    assert st == 0
    want, n_dem = _lsa_want(C, *linear_sum_assignment(C))
    assert np.array_equal(c4r, want)
    assert n_dem == 3
    _report(f"lsa {shape} {'smem' if smem else 'workspace'}", bit_exact=True, demoted=n_dem)


def _run_cascade(lib, rng, n_det, sizes, n_unconf, n_hist, all_inf=False, feat_gated=0.35):
    import ctypes as C
    from gpu_util import dev, host
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    from test_gpu_assoc import _cascade_emulated
    goff = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    n_conf = int(goff[-1])

    def costs(nr, quant, gated=0.35):
        c = rng.uniform(0, 1, (nr, n_det))
        if quant:
            c = np.round(c * quant) / quant
        c[rng.random((nr, n_det)) < gated] = INF
        if all_inf:
            c[:] = INF
        return np.ascontiguousarray(c)
    F = costs(n_conf, 16, feat_gated)
    I = costs(n_conf + n_unconf, 0)
    R = costs(n_hist, 0)
    active = (rng.random(n_conf) < 0.6).astype(np.uint8)
    conf = rng.uniform(0.3, 1.0, n_det)
    conf[0] = 0.9
    occ = (rng.random(n_det) < 0.2).astype(np.uint8)
    if all_inf:
        occ[:] = 0
    want = _cascade_emulated(F, I, R, goff, active, conf, occ, 0.5, 0.45)
    cap = max(n_conf + n_unconf, n_det, n_hist, 1)
    n_out = int(lib.fm_assoc_cascade_out_ints(cap))
    keep = [dev(a) for a in (goff, active if n_conf else np.zeros(1, np.uint8), F.reshape(-1) if F.size else np.zeros(1),
                             I.reshape(-1) if I.size else np.zeros(1), R.reshape(-1) if R.size else np.zeros(1), conf, occ)]
    sub = torch.zeros(256 * 256, dtype=torch.float64, device="cuda")
    out = torch.full((n_out,), -9, dtype=torch.int32, device="cuda")
    d = _lib.FmCascadeDesc()
    d.n_det, d.n_conf, d.n_groups, d.n_unconf, d.n_hist, d.cap = n_det, n_conf, len(sizes), n_unconf, n_hist, cap
    d.goff, d.conf_active, d.feat_cost, d.iou_cost, d.reid_cost, d.det_conf, d.det_occluded = (ptr(t) for t in keep)
    d.sub, d.out = ptr(sub), ptr(out)
    d.conf_thresh, d.max_reid_cost = 0.5, 0.45
    _lib.check(lib.fm_assoc_cascade(C.byref(d), stream_ptr()), "fm_assoc_cascade")
    o = host(out)
    assert o[0] == 0
    arr = [o[16 + k * cap: 16 + (k + 1) * cap] for k in range(14)]
    n = [int(v) for v in o[1:10]]

    def pairs(a, b, k):
        return [tuple(x) for x in zip(a[:k].tolist(), b[:k].tolist())]
    got = (pairs(arr[0], arr[1], n[0]), arr[6][:n[3]].tolist(), pairs(arr[2], arr[3], n[1]), arr[7][:n[4]].tolist(),
           pairs(arr[4], arr[5], n[2]), arr[8][:n[5]].tolist(), pairs(arr[9], arr[10], n[6]), arr[11][:n[7]].tolist(),
           arr[12][:n[8]].tolist())
    names = ("matches1", "u_trk1", "matches2", "u_trk2", "matches3", "u_trk3", "reid", "invalid", "reid_u")
    for nm, g_, w_ in zip(names, got, want):
        assert g_ == [tuple(x) if isinstance(x, (tuple, list)) else x for x in w_], (nm, g_, w_)
    assert np.array_equal(arr[13][:n_det], occ)
    return got


@pytest.mark.parametrize("case", ["n_det_256", "one_group_256", "rows_256", "hist_256", "all_256", "one_det_all_inf"])
def test_assoc_cascade_at_256(lib, case):
    """fm_assoc_cascade == the stage-by-stage emulation at the 256 limit of every dimension (n = 256 fills the
    2048-entry Numba set table) and with a single detection that every stage gates."""
    rng = np.random.default_rng(len(case))
    # feat_gated: share of FM_INF_COST appearance costs; above 0.9 many confirmed tracks find no finite pair, so that
    # the IoU stages of the active leftovers and of the unconfirmed tracks see tracks and detections
    n_det, sizes, n_unconf, n_hist, feat_gated = {
        "n_det_256": (256, [70, 50, 0, 40], 60, 50, 0.995),
        "one_group_256": (200, [256], 0, 30, 0.35),
        "rows_256": (180, [100, 0, 60], 96, 0, 0.97),
        "hist_256": (256, [40], 20, 256, 0.35),
        "all_256": (256, [256], 0, 256, 0.35),
        "one_det_all_inf": (1, [5, 0, 3], 4, 6, 0.35),
    }[case]
    got = _run_cascade(lib, rng, n_det, sizes, n_unconf, n_hist, all_inf=case == "one_det_all_inf",
                       feat_gated=feat_gated)
    if feat_gated > 0.9:
        assert got[2] and got[4]        # both IoU stages matched something
    if case == "one_det_all_inf":
        assert got[0] == [] and got[2] == [] and got[4] == [] and got[6] == []
    _report(f"cascade {case}", matches1=len(got[0]), matches2=len(got[2]), matches3=len(got[4]), reid=len(got[6]))


# ------------------------------------------------------------------------------------------------------------------
# 5. fm_feature_update
# ------------------------------------------------------------------------------------------------------------------
def _feature_model(s, cnt):
    """AverageFeature.update's average: avg = float32(float64(sum) * (1 / count)), normalised by the float32 norm,
    which is accumulated in float64 (a per-element fp32 model; only the norm's summation order is free)."""
    div = 1.0 / cnt.astype(np.float64)[:, None]
    a = (s.astype(np.float64) * div).astype(np.float32)
    nrm = np.sqrt((a.astype(np.float64) ** 2).sum(1)).astype(np.float32)
    return (a.astype(np.float64) * (1.0 / nrm.astype(np.float64))[:, None]).astype(np.float32)


@pytest.mark.parametrize("dim", [1, 100, 512, 2048])
@pytest.mark.parametrize("with_last", [False, True])
def test_feature_update_sweep(lib, dim, with_last):
    """200 scattered tracks per launch with a permuted vec_idx, counts 1 -> 50 over 50 launches (a third of the
    tracks restart at count 1 halfway); sums bit-exact, averages within 2 fp32 ulp, other slots untouched."""
    from gpu_util import dev, host
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    rng = np.random.default_rng(dim + with_last)
    cap, n, n_vec = 512, 200, 256
    slots = rng.permutation(cap)[:n].astype(np.int32)
    pools = [_sentinel32((cap, dim), t) for t in (1, 2, 3)]
    valid0 = np.full(cap, 0xAB, np.uint8)
    d_sum, d_avg, d_last = (dev(p) for p in pools)
    d_valid = dev(valid0)
    d_slots = dev(slots)
    cnt = np.zeros(n, np.int64)
    hs = np.zeros((n, dim), np.float32)
    worst = 0.
    for step in range(50):
        vec = rng.normal(size=(n_vec, dim)).astype(np.float32)
        vec /= np.linalg.norm(vec, axis=1, keepdims=True)
        vidx = rng.permutation(n_vec)[:n].astype(np.int32)
        cnt += 1
        if step == 25:
            cnt[rng.permutation(n)[:n // 3]] = 1
        d_vec, d_vidx, d_cnt = dev(vec), dev(vidx), dev(cnt.astype(np.int32))
        _lib.check(lib.fm_feature_update(ptr(d_sum), ptr(d_avg), ptr(d_last) if with_last else None, ptr(d_valid),
                                         ptr(d_slots), ptr(d_vec), ptr(d_vidx), ptr(d_cnt), n, dim, stream_ptr()),
                   "fm_feature_update")
        v = vec[vidx]
        first = cnt == 1
        hs = np.where(first[:, None], v, hs + v)
        ha = np.where(first[:, None], v, _feature_model(hs, np.maximum(cnt, 2)))
        gs, ga = host(d_sum[d_slots.long()]), host(d_avg[d_slots.long()])
        assert _same_bits(gs, hs), step
        # a sum of exactly 0 (dim 1: +1 and -1) normalises to 0 * inf = NaN in both
        nan = np.isnan(ha)
        assert np.array_equal(np.isnan(ga), nan) and (dim == 1 or not nan.any()), step
        ulp = np.spacing(np.abs(ha[~nan])).astype(np.float64)
        r = float((np.abs(ga[~nan].astype(np.float64) - ha[~nan]) / ulp).max(initial=0.))
        assert r <= 2., (step, r)
        worst = max(worst, r)
        if with_last:
            assert _same_bits(host(d_last[d_slots.long()]), v)
    other = np.ones(cap, bool)
    other[slots] = False
    got = [host(d_sum), host(d_avg), host(d_last)]
    for g, p in zip(got, pools):
        assert _same_bits(g[other], p[other])
    if not with_last:
        assert _same_bits(got[2], pools[2])
    gv = host(d_valid)
    assert np.all(gv[slots] == 1) and np.all(gv[other] == 0xAB)
    _report(f"feature_update dim={dim} last={with_last}", avg_err_ulp=worst)
