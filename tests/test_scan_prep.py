"""SURVEY 8 f-5 on the CPU: the sweep-preparation oracle (Preprocessing::cloudHandler, GLIO/src/Preprocessing.cpp:387-526) against
an independent numpy formulation, its correctly rounded atanf / atan2f against long double, and the IMU helper
(processIMU, :202-259) against a numpy restatement.  The device is checked against this oracle in test_gpu_scan_prep.py."""
import numpy as np
import pytest

from glio_b200 import synth

F, D = np.float32, np.float64
PI = np.pi


@pytest.fixture(scope="module")
def sp():
    from oracle import pyoracle_scanprep
    pyoracle_scanprep.build()
    return pyoracle_scanprep


def f_add_d(f, d):
    return (f.astype(D) + d).astype(F)


def numpy_prepare(sp, raw, n_scans):
    """Steps 1-5 for identity qIMU / q_lb, vectorised: xyz pass through unchanged, so only ring, order, time and ranges remain."""
    x, y, z = (raw[:, k].astype(F) for k in range(3))
    fin = np.isfinite(x) & np.isfinite(y) & np.isfinite(z)
    with np.errstate(invalid="ignore", over="ignore"):
        valid = fin & ~((x * x + y * y) + z * z < F(9))
    idx = np.nonzero(valid)[0]
    x, y, z = x[idx], y[idx], z[idx]
    start = -sp.cr_atan2f(y[:1], x[:1])[0]
    end = f_add_d(-sp.cr_atan2f(y[-1:], x[-1:]), 2 * PI)[0]
    if D(F(end - start)) > 3 * PI:
        end = f_add_d(np.array([end]), -2 * PI)[0]
    elif D(F(end - start)) < PI:
        end = f_add_d(np.array([end]), 2 * PI)[0]
    with np.errstate(divide="ignore", invalid="ignore"):
        a = sp.cr_atanf(z / np.sqrt(x * x + y * y)) * F(180)
    angle = (a.astype(D) / PI).astype(F)
    if n_scans == 16:
        ring = np.trunc(((angle + F(15)) / F(2)).astype(D) + 0.5).astype(int)
        ok = (ring <= 15) & (ring >= 0)
    elif n_scans == 32:
        ring = np.trunc((angle.astype(D) + 92.0 / 3.0) * 3.0 / 4.0).astype(int)
        ok = (ring <= 31) & (ring >= 0)
    else:
        hi = np.trunc((F(2) - angle).astype(D) * 3.0 + 0.5).astype(int)
        lo = 32 + np.trunc((-8.83 - angle.astype(D)) * 2.0 + 0.5).astype(int)
        ring = np.where(angle.astype(D) >= -8.83, hi, lo)
        ok = ~((angle > F(2)) | (angle.astype(D) < -24.33) | (ring > 50) | (ring < 0))
    ori = -sp.cr_atan2f(y, x)
    first = np.where(ori.astype(D) < D(start) - PI / 2, f_add_d(ori, 2 * PI), np.where(ori.astype(D) > D(start) + PI * 3 / 2, f_add_d(ori, -2 * PI), ori))
    pre = ok & ((first - start).astype(D) > PI)
    h = int(np.argmax(pre)) if pre.any() else len(ori)        # first kept point past half: the last one of the first branch
    sec = f_add_d(ori, 2 * PI)
    sec = np.where(sec.astype(D) < D(end) - PI * 3 / 2, f_add_d(sec, 2 * PI), np.where(sec.astype(D) > D(end) + PI / 2, f_add_d(sec, -2 * PI), sec))
    o = np.where(np.arange(len(ori)) <= h, first, sec)
    rel = (o - start) / F(end - start)
    inten = (ring.astype(D) + 0.1 * rel.astype(D)).astype(F)
    keep = np.nonzero(ok)[0]
    order = keep[np.argsort(ring[keep], kind="stable")]
    cloud = np.stack([x[order], y[order], z[order], inten[order]], 1)
    counts = np.bincount(ring[keep], minlength=n_scans)[:n_scans]
    before = np.concatenate([[0], np.cumsum(counts)[:-1]])
    return dict(cloud=cloud, scan_start=before + 5, scan_end=before + counts - 6, half_index=int(idx[h]) if pre.any() else -1)


@pytest.mark.parametrize("n_scans", [16, 32, 64])
def test_oracle_matches_numpy_formulation(sp, n_scans):
    s = synth.raw_sweep(n_scans)
    o = sp.prepare_scan(s["raw"], n_scans)
    ref = numpy_prepare(sp, s["raw"], n_scans)
    assert o["half_index"] == ref["half_index"] and o["half_index"] > 0     # sequential flag == first-index formulation
    assert np.array_equal(o["scan_start"], ref["scan_start"]) and np.array_equal(o["scan_end"], ref["scan_end"])
    assert np.array_equal(o["cloud"].view(np.uint32), ref["cloud"].view(np.uint32))
    assert len(o["cloud"]) > 0.8 * np.isfinite(s["raw"][:, 0]).sum() * (16 / 18 if n_scans == 16 else 0.5)


@pytest.mark.parametrize("coverage,start", [(2 * PI - 0.1, PI - 0.05), (2 * PI + 0.1, -PI + 0.05), (0.5 * PI, 0.3)])
def test_oracle_end_ori_corrections_and_half_index(sp, coverage, start):
    s = synth.raw_sweep(16, n_az=600, coverage=coverage, start_az=start)
    o = sp.prepare_scan(s["raw"], 16)
    ref = numpy_prepare(sp, s["raw"], 16)
    assert o["half_index"] == ref["half_index"]
    assert np.array_equal(o["cloud"].view(np.uint32), ref["cloud"].view(np.uint32))
    rel = (o["cloud"][:, 3] - np.floor(o["cloud"][:, 3] + 1e-6)) / 0.1
    assert rel.max() < 1.05 and rel.min() > -0.05         # both corrections keep relTime inside the sweep


def test_truncation_toward_zero_keeps_the_point(sp):
    """int() truncates toward zero: a ring value in (-1, 0) becomes ring 0 and the point is kept (:442, :449)."""
    for n_scans, elev in ((32, -92.0 / 3.0 - 0.5), (16, -16.5)):
        e = np.deg2rad(elev)
        pts = np.array([[10 * np.cos(e), 0.1, 10 * np.sin(e), 0.0], [10 * np.cos(e) * np.cos(0.3), -10 * np.cos(e) * np.sin(0.3), 10 * np.sin(e), 0.0]], np.float32)
        o = sp.prepare_scan(pts, n_scans)
        assert len(o["cloud"]) == 2 and o["scan_start"][0] == 5 and o["scan_end"][0] == 2 - 6
        assert np.floor(o["cloud"][:, 3]).max() == 0
    far = np.array([[10.0, 0.1, -10 * np.tan(np.deg2rad(33.0)), 0.0]], np.float32)     # ring value -1.75 -> -1: skipped
    assert len(sp.prepare_scan(far, 32)["cloud"]) == 0


def test_correctly_rounded_atan_against_long_double(sp):
    rng = np.random.default_rng(11)
    n = 1_000_000
    y = (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 2, n)).astype(F)
    x = (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 2, n)).astype(F)
    swp = np.concatenate([synth.raw_sweep(k)["raw"] for k in (16, 32, 64)])
    swp = swp[np.isfinite(swp[:, 0])]
    y = np.concatenate([y, swp[:, 1]]); x = np.concatenate([x, swp[:, 0]])
    with np.errstate(divide="ignore", invalid="ignore"):
        a = np.concatenate([(y / x).astype(F), swp[:, 2] / np.sqrt(swp[:, 0] * swp[:, 0] + swp[:, 1] * swp[:, 1])])
    a = a[np.isfinite(a)]
    sp.guard_hits(reset=True)
    got2 = sp.cr_atan2f(y, x)
    got1 = sp.cr_atanf(a)
    ref2 = np.arctan2(y.astype(np.longdouble), x.astype(np.longdouble)).astype(F)
    ref1 = np.arctan(a.astype(np.longdouble)).astype(F)
    assert np.array_equal(got2, ref2) and np.array_equal(got1, ref1)
    hits = sp.guard_hits()
    libm2 = int((sp.libm_atan2f(y, x) != got2).sum()); libm1 = int((sp.libm_atanf(a) != got1).sum())
    print(f"\n{len(y)} atan2f + {len(a)} atanf arguments: {hits} guard-band decisions; host libm atan2f differs from the correctly "
          f"rounded value on {libm2}, atanf on {libm1}")


def numpy_imu(state, stamps, gyro, t_cur):
    """processIMU (:222-259) with solveRotation / deltaQ, restated with numpy scalars; state = dict(idx, cur, g0, first)."""
    q = np.array([1.0, 0.0, 0.0, 0.0])
    if not state["first"]:
        if len(stamps) == 0:
            return q
        state.update(cur=stamps[0], g0=gyro[0].copy(), first=True)

    def rot(q, dt, w):
        half = (0.5 * (state["g0"] + w)) * dt / 2.0
        state["g0"] = w.copy()
        return synth.quat_mul(q, np.array([1.0, half[0], half[1], half[2]]))
    r = np.zeros(3)
    i = state["idx"]
    if i >= len(stamps):
        i -= 1                                               # quirk: step back one sample past the end
    while stamps[i] < t_cur:
        dt = stamps[i] - state["cur"]; state["cur"] = stamps[i]
        r = gyro[i].copy(); q = rot(q, dt, r)
        i += 1
        if i >= len(stamps):
            break
    if i < len(stamps):
        dt1 = t_cur - state["cur"]; dt2 = stamps[i] - t_cur
        w1 = dt2 / (dt1 + dt2); w2 = dt1 / (dt1 + dt2)
        r = w1 * r + w2 * gyro[i]                            # quirk: r is 0 when no sample was consumed in this call
        q = rot(q, dt1, r)
    state["cur"] = t_cur; state["idx"] = i
    return np.array([1.0, 0.0, 0.0, 0.0]) if np.isnan(q).any() else q      # :415-417


def test_imu_helper_against_numpy(sp):
    rng = np.random.default_rng(3)
    stamps = 10.0 + np.arange(80) / 400.0
    gyro = rng.normal(0.0, 0.3, (80, 3))
    st = sp.ImuState(); ref = dict(idx=0, cur=-1.0, g0=np.zeros(3), first=False)
    assert np.array_equal(sp.imu_sweep_rotation(st, stamps[:0], gyro[:0], 9.0), [1, 0, 0, 0])    # no sample yet
    # 9.999: before the first sample (0 / 0 weights -> NaN -> identity); 10.0001: no sample consumed after the first (the
    # interpolation mixes r = 0 with the next sample); then ordinary sweeps; then two calls past the end of the buffer (index
    # steps back one sample)
    for t in (9.999, 10.0001, 10.05, 10.1, 10.1001, 10.3, 10.4):
        with np.errstate(divide="ignore", invalid="ignore"):
            q = sp.imu_sweep_rotation(st, stamps, gyro, t)
            qr = numpy_imu(ref, stamps, gyro, t)
        assert np.array_equal(q, qr), (t, q, qr)
        assert st.idx_imu == ref["idx"] and st.current_time_imu == ref["cur"]
    assert st.idx_imu == len(stamps) and not np.array_equal(q, [1, 0, 0, 0])


def test_imu_helper_matches_oracle(sp):
    """The library's host helper (glio_imu_sweep_rotation) against the oracle's, state included (the sample before the buffer
    leaves a NaN gyr_0 behind, as in the reference)."""
    from glio_b200 import api
    s = synth.raw_sweep(16, n_az=10, yaw_rate=0.7)
    rng = np.random.default_rng(5)
    gyro = s["gyro"] + rng.normal(0, 0.05, s["gyro"].shape)
    stamps = s["stamps"]
    a, b = api.ImuState(), sp.ImuState()
    for t in (stamps[0] - 0.01, stamps[10] + 0.001, stamps[40], stamps[-1] + 0.05, stamps[-1] + 0.1):
        with np.errstate(divide="ignore", invalid="ignore"):
            qa = api.imu_sweep_rotation(a, stamps, gyro, t)
            qb = sp.imu_sweep_rotation(b, stamps, gyro, t)
        assert np.array_equal(qa, qb), (t, qa, qb)
        assert a.idx_imu == b.idx_imu and a.current_time_imu == b.current_time_imu and np.array_equal(list(a.gyr_0), list(b.gyr_0), equal_nan=True)
