"""SURVEY 8 f-5 on the device: glio_prepare_scan (Preprocessing::cloudHandler, GLIO/src/Preprocessing.cpp:387-526) against the
sequential CPU oracle.  Identity qIMU: every output bit for bit.  Rotating sensor: everything bit for bit except xyz, which may
differ by one float ulp (device double sin against libm sin in Eigen's slerp)."""
import numpy as np
import pytest

from glio_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sp():
    from oracle import pyoracle_scanprep
    pyoracle_scanprep.build()
    return pyoracle_scanprep


@pytest.fixture(scope="module")
def ctx():
    from glio_b200 import api
    c = api.Context(0)
    yield c
    c.close()


_SWEEPS = {}


def sweep(n_rings, **kw):
    key = (n_rings, tuple(sorted(kw.items())))
    if key not in _SWEEPS:
        _SWEEPS[key] = synth.raw_sweep(n_rings, **kw)
    return _SWEEPS[key]


def as_stride(raw4, stride):
    if stride == 4:
        return np.ascontiguousarray(raw4)
    buf = np.full((len(raw4), 8), np.nan, np.float32)        # pcl::PointXYZI: x y z 1 | intensity pad pad pad
    buf[:, :3] = raw4[:, :3]; buf[:, 3] = 1.0; buf[:, 4] = raw4[:, 3]
    return buf


def run_device(ctx, raw, n_scans, q_imu, mem, out):
    import torch
    arg = torch.from_numpy(raw).cuda() if mem == "device" else raw
    cloud, ss, se = ctx.prepare_scan(arg, n_scans, q_imu=q_imu, out=out)
    if out == "device":
        assert cloud.is_cuda
        cloud = cloud.cpu().numpy()
    return cloud, ss, se


def ulp_diff(a, b):
    ia = a.view(np.int32).astype(np.int64); ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia); ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.abs(ia - ib)


def check(d, o, exact_xyz=True):
    cloud, ss, se = d
    assert cloud.shape == o["cloud"].shape, (cloud.shape, o["cloud"].shape)
    assert np.array_equal(ss, o["scan_start"]) and np.array_equal(se, o["scan_end"])
    assert np.array_equal(cloud[:, 3].view(np.uint32), o["cloud"][:, 3].view(np.uint32)), "intensity / order differs"
    if exact_xyz:
        assert np.array_equal(cloud[:, :3].view(np.uint32), o["cloud"][:, :3].view(np.uint32)), "xyz differs"
    else:
        u = ulp_diff(cloud[:, :3], o["cloud"][:, :3])
        assert u.max() <= 1, f"xyz differs by up to {u.max()} ulp; {int((u > 0).sum())} of {u.size} coordinates not identical"


@pytest.mark.parametrize("n_scans", [16, 32, 64])
@pytest.mark.parametrize("stride", [4, 8])
@pytest.mark.parametrize("mem,out", [("host", "host"), ("device", "device"), ("host", "device"), ("device", "host")])
def test_prepare_scan_identity_imu_bit_exact(sp, ctx, n_scans, stride, mem, out):
    s = sweep(n_scans)
    raw = as_stride(s["raw"], stride)
    o = sp.prepare_scan(raw, n_scans, None, synth.Q_LB)
    check(run_device(ctx, raw, n_scans, None, mem, out), o)


@pytest.mark.parametrize("n_scans", [16, 32, 64])
@pytest.mark.parametrize("stride", [4, 8])
def test_prepare_scan_rotating_sensor(sp, ctx, n_scans, stride):
    s = sweep(n_scans, yaw_rate=0.8)
    st = sp.ImuState()
    q = sp.imu_sweep_rotation(st, s["stamps"], s["gyro"], s["t_scan_next"])
    assert abs(q[3]) > 0.01
    raw = as_stride(s["raw"], stride)
    o = sp.prepare_scan(raw, n_scans, q, synth.Q_LB)
    check(run_device(ctx, raw, n_scans, q, "host", "host"), o, exact_xyz=False)


def test_prepare_scan_rotating_extrinsic(sp, ctx):
    """A non-identity q_lb (the conjugation of :191 no longer cancels) with a rotating sensor."""
    s = sweep(32, yaw_rate=-0.6)
    q = sp.imu_sweep_rotation(sp.ImuState(), s["stamps"], s["gyro"], s["t_scan_next"])
    q_lb = synth.quat_from_rpy(0.02, -0.01, 0.3)
    o = sp.prepare_scan(s["raw"], 32, q, q_lb)
    d = ctx.prepare_scan(s["raw"], 32, q_imu=q, q_lb=q_lb)
    check(d, o, exact_xyz=False)


def test_guard_band_counter(sp, ctx):
    """The double-double decision is taken now and then on a full sweep, and its results still match the oracle bit for bit."""
    ctx.scanprep_guard_hits(reset=True)
    hits = 0
    for seed in range(3):
        s = synth.raw_sweep(64, seed=1000 + seed, n_az=2000)
        o = sp.prepare_scan(s["raw"], 64)
        check(ctx.prepare_scan(s["raw"], 64), o)
    hits = ctx.scanprep_guard_hits()
    assert hits > 0
    assert ctx.scanprep_guard_hits(reset=True) == hits and ctx.scanprep_guard_hits() == 0


@pytest.mark.parametrize("rotating", [False, True])
def test_prepare_then_extract_on_device(sp, oracle, ctx, rotating):
    s = sweep(32, yaw_rate=0.8 if rotating else 0.0)
    q = sp.imu_sweep_rotation(sp.ImuState(), s["stamps"], s["gyro"], s["t_scan_next"]) if rotating else None
    o = sp.prepare_scan(s["raw"], 32, q, synth.Q_LB)
    cloud, ss, se = ctx.prepare_scan(s["raw"], 32, q_imu=q, out="device")
    d = ctx.extract_features(cloud, ss, se, ds_rate=1, edge_thres=1.0, surf_thres=0.1, ds_v=0.4)
    # identity qIMU: the oracle's own cloud; rotating: the device's cloud (xyz may differ by an ulp from the oracle's)
    ref_cloud = o["cloud"] if not rotating else cloud.cpu().numpy()
    if not rotating:
        assert np.array_equal(cloud.cpu().numpy().view(np.uint32), o["cloud"].view(np.uint32))
    e = oracle.extract_features(ref_cloud, ss, se, ds_rate=1, edge_thres=1.0, surf_thres=0.1, ds_v=0.4, stable=True)
    assert np.array_equal(d["curvature"], e["curvature"]) and np.array_equal(d["label"], e["label"])
    for k in ("sharp", "less_sharp", "flat", "less_flat"):
        assert np.array_equal(d[k], e[k]), k
    assert np.array_equal(d["less_flat_ds"], e["less_flat_ds"])
    assert len(d["sharp"]) > 20 and len(d["flat"]) > 200


# ---- edge cases ---------------------------------------------------------------------------------------------------------

def test_everything_filtered_is_an_error_and_context_stays_usable(sp, ctx):
    from glio_b200 import api
    raw = np.zeros((100, 4), np.float32)
    raw[::2, :3] = np.nan
    raw[1::2, :3] = [1.0, 1.0, 1.0]                          # closer than 3 m
    with pytest.raises(api.GlioError, match="finite"):
        ctx.prepare_scan(raw, 32)
    with pytest.raises(ValueError):
        sp.prepare_scan(raw, 32)
    with pytest.raises(api.GlioError, match="n_scans"):
        ctx.prepare_scan(sweep(32)["raw"], 40)
    s = sweep(32)
    check(ctx.prepare_scan(s["raw"], 32), sp.prepare_scan(s["raw"], 32))


def test_one_kept_point_and_only_skipped_rings(sp, ctx):
    raw = np.array([[10.0, 0.5, -0.3, 5.0], [np.nan, 0, 0, 0], [0.1, 0.2, 0.3, 1.0]], np.float32)
    for n_scans in (16, 32, 64):
        o = sp.prepare_scan(raw, n_scans)
        d = ctx.prepare_scan(raw, n_scans)
        assert len(o["cloud"]) == 1
        check(d, o)
    up = np.array([[10.0, 0.5, 9.0, 0.0]] * 3, np.float32)        # 42 degrees up: every ring rule skips it
    for n_scans in (16, 32, 64):
        o = sp.prepare_scan(up, n_scans)
        d = ctx.prepare_scan(up, n_scans)
        assert len(o["cloud"]) == 0 and len(d[0]) == 0
        check(d, o)


def test_half_passed_never(sp, ctx):
    s = synth.raw_sweep(16, n_az=400, coverage=0.5 * np.pi)     # a quarter turn: no point gets past startOri + pi
    o = sp.prepare_scan(s["raw"], 16)
    assert o["half_index"] == -1
    check(ctx.prepare_scan(s["raw"], 16), o)


def test_half_passed_set_at_first_processed_point(sp, ctx):
    """startOri comes from the first point left after the NaN / 3 m filters even when its ring is skipped; the next kept point can
    then be past half at once."""
    head = np.array([[10.0, -0.01, 30.0, 0.0],               # 71 degrees up: ring skipped, startOri ~ +0.001
                     [-10.0, 0.5, -0.3, 0.0]], np.float32)   # first kept point, azimuth ~ pi from it
    s = synth.raw_sweep(32, n_az=300)
    raw = np.concatenate([head, s["raw"]])
    o = sp.prepare_scan(raw, 32)
    assert o["half_index"] == 1
    check(ctx.prepare_scan(raw, 32), o)


def test_64_lines_rejected_rings_and_z_axis(sp, ctx):
    s = sweep(64)
    o = sp.prepare_scan(s["raw"], 64)
    ss, se = o["scan_start"], o["scan_end"]
    assert (se[51:] - ss[51:] == -11).all()                  # rings 51..63 are empty: start = end + 11
    z = np.isfinite(s["raw"][:, 0]) & (s["raw"][:, 0] == 0) & (s["raw"][:, 1] == 0)
    assert z.sum() > 0
    check(ctx.prepare_scan(s["raw"], 64), o)


def test_nan_q_imu_is_identity(sp, ctx):
    s = sweep(16)
    q = np.array([np.nan, 0.0, 0.0, 0.1])
    o = sp.prepare_scan(s["raw"], 16, None)
    check(ctx.prepare_scan(s["raw"], 16, q_imu=q), o)


def test_out_capacity_too_small(sp, ctx):
    import ctypes as C
    import torch
    from glio_b200 import api
    s = sweep(16)
    raw = np.ascontiguousarray(s["raw"])
    m = len(sp.prepare_scan(raw, 16)["cloud"])
    L = api.lib()
    for out_mem in (api.HOST, api.DEVICE):
        cap = m - 7
        sentinel = np.float32(-1234.5)
        if out_mem == api.HOST:
            buf = np.full((cap + 16, 4), sentinel, np.float32); ptr = buf.ctypes.data_as(C.c_void_p)
        else:
            tb = torch.full((cap + 16, 4), float(sentinel), dtype=torch.float32, device="cuda"); ptr = C.c_void_p(tb.data_ptr())
        n_out = C.c_int64(0)
        ss = np.zeros(16, np.int32); se = np.zeros(16, np.int32)
        rc = L.glio_prepare_scan(ctx._h, raw.ctypes.data_as(C.c_void_p), C.c_int64(len(raw)), C.c_int(4), C.c_int(api.HOST), C.c_int(16),
                                 None, None, ptr, C.c_int(out_mem), C.c_int64(cap), C.byref(n_out),
                                 ss.ctypes.data_as(C.c_void_p), se.ctypes.data_as(C.c_void_p))
        assert rc == -3 and n_out.value == m
        after = buf if out_mem == api.HOST else tb.cpu().numpy()
        assert (after[cap:] == sentinel).all(), "write past out_capacity"
    check(ctx.prepare_scan(raw, 16), sp.prepare_scan(raw, 16))


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 255, 256, 257, 1000, 4097, 65537, 130000])
def test_sizes(sp, ctx, n):
    base = sweep(64, n_az=2100)["raw"]
    assert len(base) >= 130000
    raw = np.ascontiguousarray(base[:n])
    raw[0, :3] = [12.0, 3.0, -1.0]                           # a valid first point for every size
    o = sp.prepare_scan(raw, 64)
    check(ctx.prepare_scan(raw, 64), o)


@pytest.mark.parametrize("coverage,start", [(2 * np.pi - 0.1, np.pi - 0.05), (2 * np.pi + 0.1, -np.pi + 0.05), (2 * np.pi - 0.02, 0.3)])
def test_end_ori_corrections(sp, ctx, coverage, start):
    s = synth.raw_sweep(16, n_az=800, coverage=coverage, start_az=start, nan_frac=0.0, near_frac=0.0, n_zaxis=0)
    check(ctx.prepare_scan(s["raw"], 16), sp.prepare_scan(s["raw"], 16))


def _raw_call(ctx, raw_ptr, n, mem, out_ptr, out_mem, cap):
    import ctypes as C
    from glio_b200 import api
    n_out = C.c_int64(-1)
    ss = np.zeros(32, np.int32); se = np.zeros(32, np.int32)
    rc = api.lib().glio_prepare_scan(ctx._h, raw_ptr, C.c_int64(n), C.c_int(4), C.c_int(mem), C.c_int(32), None, None, out_ptr,
                                     C.c_int(out_mem), C.c_int64(cap), C.byref(n_out), ss.ctypes.data_as(C.c_void_p),
                                     se.ctypes.data_as(C.c_void_p))
    return rc, n_out.value


def test_bad_device_pointers_are_argument_errors(sp, ctx):
    """Misaligned device output (float4 stores), misaligned raw input and a host pointer declared GLIO_DEVICE are rejected before
    anything is launched; the context keeps working afterwards."""
    import ctypes as C
    import torch
    from glio_b200 import api
    s = sweep(32)
    raw = np.ascontiguousarray(s["raw"]); n = len(raw)
    hraw = raw.ctypes.data_as(C.c_void_p)
    out = torch.zeros((n + 1, 4), dtype=torch.float32, device="cuda")
    assert out.data_ptr() % 16 == 0
    rc, m = _raw_call(ctx, hraw, n, api.HOST, C.c_void_p(out.data_ptr() + 4), api.DEVICE, n)          # float* + 1
    assert rc == -3 and m == -1 and "16-byte" in api.lib().glio_last_error(ctx._h).decode()
    draw = torch.from_numpy(raw).cuda()
    craw = torch.zeros(n * 4 + 1, dtype=torch.float32, device="cuda")
    rc, _ = _raw_call(ctx, C.c_void_p(draw.data_ptr() + 2), n, api.DEVICE, C.c_void_p(out.data_ptr()), api.DEVICE, n)
    assert rc == -3 and "4-byte" in api.lib().glio_last_error(ctx._h).decode()
    rc, _ = _raw_call(ctx, hraw, n, api.DEVICE, C.c_void_p(out.data_ptr()), api.DEVICE, n)            # host memory as GLIO_DEVICE
    assert rc == -3 and "not device memory" in api.lib().glio_last_error(ctx._h).decode()
    hout = np.zeros((n, 4), np.float32)
    rc, _ = _raw_call(ctx, hraw, n, api.HOST, hout.ctypes.data_as(C.c_void_p), api.DEVICE, n)
    assert rc == -3 and "not device memory" in api.lib().glio_last_error(ctx._h).decode()
    assert (out == 0).all() and (craw == 0).all()
    check(run_device(ctx, raw, 32, None, "host", "device"), sp.prepare_scan(raw, 32))


@pytest.mark.skipif("__import__('torch').cuda.device_count() < 2")
def test_memory_of_another_gpu_is_an_argument_error(sp):
    import ctypes as C
    import torch
    from glio_b200 import api
    ctx1 = api.Context(1)
    try:
        raw = np.ascontiguousarray(sweep(32)["raw"]); n = len(raw)
        out0 = torch.zeros((n, 4), dtype=torch.float32, device="cuda:0")
        rc, _ = _raw_call(ctx1, raw.ctypes.data_as(C.c_void_p), n, api.HOST, C.c_void_p(out0.data_ptr()), api.DEVICE, n)
        assert rc == -3 and "context's GPU" in api.lib().glio_last_error(ctx1._h).decode()
        with torch.cuda.device(0):                       # torch's current device differs from the context's: still allocated on GPU 1
            cloud, _, _ = ctx1.prepare_scan(raw, 32, out="device")
        assert cloud.device == torch.device("cuda", 1)
        check((cloud.cpu().numpy(),) + tuple(ctx1.prepare_scan(raw, 32)[1:]), sp.prepare_scan(raw, 32))
    finally:
        ctx1.close()
