"""Edge cases of the residual-evaluation kernels (K2 unary plane, K2b binary plane, K2e point-to-edge) against the
extended-precision reference of tests/eval_reference.py, within its a-priori bound, and against the oracle at the 1e-11
parity bar where the oracle is affordable and the fixture stays near the origin.

Inputs go in through the C ABI's own upload paths (set_matches, batch_set_pair_matches, set_edges), so every residual count
and therefore every work-item plan is exact.  The cases cover the work-item boundaries of plan_items and the kernels' software
pipeline / 8-wide partial sums, windows on both sides of the by-value pose limit (EV_MAXW = 64), non-unit quaternions, w = 0,
kilometre offsets, the Huber edges, a NaN in one keyframe, and the state the evaluations share across calls."""
import numpy as np
import pytest

from tests import eval_reference as er

pytestmark = pytest.mark.gpu

REL = 1e-11
ITEM_MAX = 2048           # GLIO_ITEM_MAX
EV_MAXW = 64
Q_LB, T_LB = er.Q_LB_NONUNIT, er.T_LB
EXCESS = {}               # factor -> largest |device - reference| / (2^-53 M) seen


def _note(factor, e):
    EXCESS[factor] = max(EXCESS.get(factor, 0.0), e)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nlargest |device - reference| / (2^-53 M) per factor (bound %d): %s"
          % (er.KAPPA, ", ".join(f"{k} {v:.3g}" for k, v in sorted(EXCESS.items()))))


def _ctx(**kw):
    from glio_b200 import api
    kw.setdefault("q_lb", Q_LB); kw.setdefault("t_lb", T_LB)
    return api.Context(0, **kw)


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def plan_items(counts, eval_slots):
    """plan_items of capi.cu: (item size, per-keyframe list of item counts)."""
    n_total = sum(counts)
    item = -(-n_total // max(eval_slots, 1))
    item = max(ITEM_MAX, -(-item // 256) * 256)
    plan = []
    for n in counts:
        parts = max(1, -(-n // item))
        per = -(-(-(-n // parts)) // 256) * 256
        plan.append([min(per, n - o) for o in range(0, n, per)])
    return item, plan


def _upload(ctx, per_kf):
    for k, m in enumerate(per_kf):
        if m is None:
            ctx.set_matches(k, np.zeros((0, 3), np.float32), np.zeros((0, 4), np.float32), np.zeros(0, np.float32))
        else:
            ctx.set_matches(k, m["cp"], m["nsd"], m["weight"])


def _unary_fixture(rng, poses, counts, **kw):
    return [er.make_unary(rng, poses[k], n, Q_LB, T_LB, **kw) if n else None for k, n in enumerate(counts)]


def _check_unary(ctx, poses, per_kf, jac_kind=0, huber=1.0, unit_score=False, nonvacuous=False, factor="unary"):
    lc = ctx.params.lidar_const
    R = er.unary_blocks(poses, per_kf, Q_LB, T_LB, lc, huber, jac_kind=jac_kind, unit_score=unit_score)
    d = ctx.eval_unary(poses, jac_kind=jac_kind)
    _note(factor, er.assert_within(d["H"], R["H"], R["MH"], f"{factor} H"))
    _note(factor, er.assert_within(d["g"], R["g"], R["Mg"], f"{factor} g"))
    _note(factor, er.assert_within(d["cost"], R["cost"], R["Mcost"], f"{factor} cost"))
    c = ctx.eval_unary(poses, want_jac=False)["cost"]
    _note(factor, er.assert_within(c, R["cost"], R["Mcost"], f"{factor} cost-only"))
    if nonvacuous:
        # the bound must be far below the blocks' scale, or it would pass a dropped residual
        for k in range(len(poses)):
            if np.max(np.abs(R["H"][k])) > 0:
                assert er.KAPPA * er.U * np.max(R["MH"][k]) < 1e-9 * np.max(np.abs(R["H"][k]))
    return d, R


def _oracle_unary(oracle, ctx, poses, per_kf, jac_kind=0, huber=1.0):
    ks = [k for k, m in enumerate(per_kf) if m is not None]
    kf = np.concatenate([np.full(len(per_kf[k]["cp"]), k, np.int32) for k in ks])
    cp = np.concatenate([per_kf[k]["cp"] for k in ks]); nsd = np.concatenate([per_kf[k]["nsd"] for k in ks])
    score = ctx.params.lidar_const * np.concatenate([per_kf[k]["weight"] for k in ks]).astype(np.float64)
    return oracle.eval_unary(poses, Q_LB, T_LB, kf, cp, nsd, score, huber_delta=huber, mode=0, jac_kind=jac_kind), kf


def _assert_oracle(o, kf, d, W):
    for k in range(W):
        Hk = o["H"][6 * k:6 * k + 6, 6 * k:6 * k + 6]
        assert np.max(np.abs(d["H"][k] - Hk)) <= REL * max(np.max(np.abs(Hk)), 1e-300)
        gk = o["g"][6 * k:6 * k + 6]
        assert np.max(np.abs(d["g"][k] - gk)) <= REL * max(np.max(np.abs(gk)), 1e-300)
        ck = o["cost"][kf == k].sum()
        assert abs(d["cost"][k] - ck) <= REL * abs(ck)


# ---------------------------------------------------------------------------------------------------------------------------
# K2: work-item shapes
# ---------------------------------------------------------------------------------------------------------------------------
ITEM_COUNTS = [1, 200, 255, 256, 257, 511, 512, 513, 1025, 2047, 2048, 14336, 16384, 18432, 32768, 34816, 16385]


def test_unary_item_shapes(oracle):
    """One keyframe per count: single items of 1..2048 residuals (c mod 512 in {0, 1, 255, 256, 257, 511}), keyframes of
    7, 8, 9, 16, 17 items and a last item of one residual (n = 16385)."""
    rng = np.random.default_rng(101)
    item, plan = plan_items(ITEM_COUNTS, 2 * _sms())
    assert item == ITEM_MAX
    nitems = [len(p) for p in plan]
    assert {7, 8, 9, 16, 17} <= set(nitems)
    assert plan[ITEM_COUNTS.index(16385)][-1] == 1
    assert {c % 512 for c in ITEM_COUNTS if c <= ITEM_MAX} >= {0, 1, 255, 256, 257, 511}
    W = len(ITEM_COUNTS)
    poses = er.make_poses(W, rng)
    per = _unary_fixture(rng, poses, ITEM_COUNTS)
    ctx = _ctx()
    try:
        _upload(ctx, per)
        for jk in (0, 1):
            d, R = _check_unary(ctx, poses, per, jac_kind=jk, nonvacuous=True)
            o, kf = _oracle_unary(oracle, ctx, poses, per, jac_kind=jk)
            _assert_oracle(o, kf, d, W)
    finally:
        ctx.close()


def test_unary_item_size_above_2048():
    """A window of more than 2048 x 2 x SMs residuals: items grow past GLIO_ITEM_MAX (256-aligned)."""
    rng = np.random.default_rng(102)
    cap = ITEM_MAX * 2 * _sms()
    counts = [cap // 4 + 9001, cap // 4 + 1, 300, cap // 4 + 4097, cap // 4 + 77]
    item, plan = plan_items(counts, 2 * _sms())
    assert item > ITEM_MAX and item % 256 == 0 and sum(counts) > cap
    assert max(len(p) for p in plan) > 16
    poses = er.make_poses(len(counts), rng)
    per = _unary_fixture(rng, poses, counts)
    ctx = _ctx()
    try:
        _upload(ctx, per)
        _check_unary(ctx, poses, per, nonvacuous=True)
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------
# K2: window sizes around the by-value pose limit, empty keyframes
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [1, 63, 64, 65, 130, 4096])
def test_unary_window_sizes(oracle, W):
    rng = np.random.default_rng(200 + W)
    n_per = 20 if W == 4096 else 300
    counts = [int(rng.integers(n_per // 2, 2 * n_per)) for _ in range(W)]
    if W >= 3:
        counts[0] = counts[-1] = 0                 # empty first and last keyframes
    if W >= 63:
        counts[W // 2:W // 2 + 5] = [0] * 5        # a run of empty keyframes
    poses = er.make_poses(W, rng)
    per = _unary_fixture(rng, poses, counts)
    ctx = _ctx()
    try:
        _upload(ctx, per)
        for jk in (0, 1):
            d, R = _check_unary(ctx, poses, per, jac_kind=jk, nonvacuous=True)
            if W <= 70:
                o, kf = _oracle_unary(oracle, ctx, poses, per, jac_kind=jk)
                _assert_oracle(o, kf, d, W)
            empty = [k for k, n in enumerate(counts) if n == 0]
            assert all(not d["H"][k].any() and not d["g"][k].any() and d["cost"][k] == 0 for k in empty)
    finally:
        ctx.close()


def test_unary_empty_window_then_evaluation():
    """A window without residuals returns zeros (nothing is launched); the next, non-empty evaluation is unaffected."""
    rng = np.random.default_rng(210)
    for W in (3, 65):
        poses = er.make_poses(W, rng)
        ctx = _ctx()
        try:
            _upload(ctx, [None] * W)
            for jk in (0, 1):
                d = ctx.eval_unary(poses, jac_kind=jk)
                assert not d["H"].any() and not d["g"].any() and not d["cost"].any()
            assert not ctx.eval_unary(poses, want_jac=False)["cost"].any()
            per = _unary_fixture(rng, poses, [0] + [700] * (W - 1))
            _upload(ctx, per)
            _check_unary(ctx, poses, per)
        finally:
            ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------
# K2: pose and parameter edges
# ---------------------------------------------------------------------------------------------------------------------------
def test_unary_km_offsets_mixed():
    """3 km and 20 km from the origin in one window (n.(a+t) + d cancels two terms of ~1e4): the reference bound is the bar."""
    rng = np.random.default_rng(301)
    offs = np.array([0.0, 3000.0, 20000.0, 3000.0, 20000.0, 50.0] * 12)   # 72 keyframes: the device-pose path
    for W in (6, 72):
        poses = er.make_poses(W, rng, offset=offs[:W])
        per = _unary_fixture(rng, poses, [int(rng.integers(200, 3000)) for _ in range(W)])
        ctx = _ctx()
        try:
            _upload(ctx, per)
            for jk in (0, 1):
                _check_unary(ctx, poses, per, jac_kind=jk)
        finally:
            ctx.close()


@pytest.mark.parametrize("case", ["q_lb_nonunit", "w_zero", "q_norm_half_two_ambient"])
def test_unary_quaternion_edges(oracle, case):
    """Non-unit q_lb (Eigen inverse = conj / |q|^2), 180-degree poses (w = 0), and pose quaternions of norm 0.5 and 2 with the
    ambient columns of the marginalisation (jac_kind 1)."""
    rng = np.random.default_rng({"q_lb_nonunit": 302, "w_zero": 303, "q_norm_half_two_ambient": 304}[case])
    W = 8
    if case == "q_norm_half_two_ambient":
        poses = er.make_poses(W, rng, qnorm=[0.5, 2.0] * (W // 2)); kinds = (1,)
    else:
        poses = er.make_poses(W, rng, w_zero=(case == "w_zero")); kinds = (0, 1)
    per = _unary_fixture(rng, poses, [int(rng.integers(300, 2500)) for _ in range(W)])
    ctx = _ctx()
    try:
        _upload(ctx, per)
        for jk in kinds:
            d, R = _check_unary(ctx, poses, per, jac_kind=jk, nonvacuous=True)
            o, kf = _oracle_unary(oracle, ctx, poses, per, jac_kind=jk)
            _assert_oracle(o, kf, d, W)
    finally:
        ctx.close()


@pytest.mark.xfail(strict=True, reason="the tangent rotation columns use R(q)p_b; Ceres' [1,d](x)q gives q p_b q* = R(q)p_b - (1-|q|^2) p_b, "
                                       "which differs when |q| != 1")
def test_unary_tangent_nonunit_pose_quaternion():
    rng = np.random.default_rng(311)
    W = 4
    poses = er.make_poses(W, rng, qnorm=[0.5, 2.0, 0.5, 2.0])
    per = _unary_fixture(rng, poses, [1000] * W)
    ctx = _ctx()
    try:
        _upload(ctx, per)
        _check_unary(ctx, poses, per, jac_kind=0)
    finally:
        ctx.close()


@pytest.mark.parametrize("huber", [0.0, 1e-6])
def test_unary_huber_edges(oracle, huber):
    """huber_delta = 0 (no loss) and a delta so small that every residual is in the Huber region."""
    rng = np.random.default_rng(320)
    W = 5
    poses = er.make_poses(W, rng)
    per = _unary_fixture(rng, poses, [257, 1025, 2049, 511, 4096])
    ctx = _ctx(huber_delta=huber)
    try:
        _upload(ctx, per)
        for jk in (0, 1):
            # with a tiny delta even near-zero residuals are outliers, and sqrt(delta/|r|) of those is ill-conditioned: no
            # non-vacuity check for that case
            d, R = _check_unary(ctx, poses, per, jac_kind=jk, huber=huber, nonvacuous=(huber == 0.0))
            o, kf = _oracle_unary(oracle, ctx, poses, per, jac_kind=jk, huber=huber)
            if huber == 0.0:
                _assert_oracle(o, kf, d, W)     # for the tiny delta the same conditioning puts two fp64 results ~1e-9 apart
            else:
                assert np.all(np.abs(o["r"]) > huber)       # |r_corrected| = sqrt(delta |r|) > delta: every residual is an outlier
    finally:
        ctx.close()


def test_unary_scores_zero_weights_and_zero_residuals():
    """unit_score = 1 (score = lidar_const), zero weights, and residuals that are exactly zero."""
    rng = np.random.default_rng(330)
    W = 4
    poses = er.make_poses(W, rng)
    per = [er.make_unary(rng, poses[k], 1500, Q_LB, T_LB, zero_weight_frac=0.3, exact_zero=200) for k in range(W)]
    per.append(er.make_unary(rng, er.make_poses(1, rng)[0], 300, Q_LB, T_LB, exact_zero=300))     # a keyframe of zeros only
    poses = np.concatenate([poses, er.make_poses(1, rng)])
    for unit in (0, 1):
        ctx = _ctx(unit_score=unit)
        try:
            _upload(ctx, per)
            for jk in (0, 1):
                d, _ = _check_unary(ctx, poses, per, jac_kind=jk, unit_score=bool(unit), nonvacuous=True)
            assert not d["H"][W].any() and not d["g"][W].any() and d["cost"][W] == 0.0
        finally:
            ctx.close()


def test_unary_nan_stays_in_its_keyframe():
    """A NaN in one keyframe's nsd makes that keyframe's cost non-finite (solve_core relies on it reaching the host); every
    other keyframe's block is bit-identical to the run without it."""
    rng = np.random.default_rng(340)
    for W in (6, 66):
        poses = er.make_poses(W, rng)
        per = _unary_fixture(rng, poses, [int(rng.integers(300, 5000)) for _ in range(W)])
        ctx = _ctx()
        try:
            _upload(ctx, per)
            base = [ctx.eval_unary(poses, jac_kind=jk) for jk in (0, 1)]
            base_c = ctx.eval_unary(poses, want_jac=False)["cost"]
            bad = W // 2
            m = dict(per[bad]); m["nsd"] = m["nsd"].copy(); m["nsd"][len(m["nsd"]) // 2, 3] = np.nan
            ctx.set_matches(bad, m["cp"], m["nsd"], m["weight"])
            others = np.arange(W) != bad
            for jk in (0, 1):
                d = ctx.eval_unary(poses, jac_kind=jk)
                assert not np.isfinite(d["cost"][bad])
                for key in ("H", "g", "cost"):
                    assert np.array_equal(d[key][others], base[jk][key][others])
            c = ctx.eval_unary(poses, want_jac=False)["cost"]
            assert not np.isfinite(c[bad]) and np.array_equal(c[others], base_c[others])
        finally:
            ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------
# per-residual path
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 255, 256, 257])
def test_unary_per_residual_counts(n):
    rng = np.random.default_rng(400 + n)
    poses = np.concatenate([er.make_poses(1, rng), er.make_poses(1, rng, offset=20000.0), er.make_poses(1, rng, qnorm=2.0)])
    ctx = _ctx()
    try:
        for i, pose in enumerate(poses):
            m = er.make_unary(rng, pose, n, Q_LB, T_LB)
            ctx.set_matches(2, m["cp"], m["nsd"], m["weight"])
            kinds = (1,) if i == 2 else (0, 1)          # |q| = 2: the ambient columns only (see the xfail above)
            for jk in kinds:
                r, J = ctx.eval_unary_residuals(2, pose, n, jac_kind=jk)
                R = er.unary_residuals(pose, m["cp"], m["nsd"], m["weight"], Q_LB, T_LB, ctx.params.lidar_const, 1.0, jac_kind=jk)
                assert len(r) == n
                _note("unary r/J", er.assert_within(r, R["r"], R["Mr"], "r"))
                _note("unary r/J", er.assert_within(J, R["J"], R["MJ"], "J"))
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------
# state across calls
# ---------------------------------------------------------------------------------------------------------------------------
def test_state_across_calls():
    """Repeated calls are bit-identical; W -> W' -> W re-plans the items and reproduces the first result; unary, edge and binary
    evaluations interleave (unary and edge share the ticket) and cost-only alternates with Jacobian evaluations."""
    rng = np.random.default_rng(500)
    W, W2 = 70, 12
    poses = er.make_poses(W, rng)
    per = _unary_fixture(rng, poses, [int(rng.integers(100, 4000)) for _ in range(W)])
    edges = [er.make_edges(rng, poses[k], int(rng.integers(100, 3000)), Q_LB, T_LB) for k in range(W2)]
    ctx = _ctx()
    try:
        _upload(ctx, per)
        for k, e in enumerate(edges):
            ctx.set_edges(k, e["cp"], e["pa"], e["pb"], e["s"])
        pairs = [(1, 0), (0, 1), (3, 7)]
        for cur, oth in pairs:
            m = er.make_pair(rng, poses[cur], poses[oth], 3000)
            ctx.batch_set_pair_matches(cur, oth, m["cp"], m["nc"], m["weight"])
        first = [ctx.eval_unary(poses, jac_kind=jk) for jk in (0, 1)]
        first_c = ctx.eval_unary(poses, want_jac=False)["cost"]
        first_e = ctx.eval_edge(poses[:W2]); first_b = ctx.eval_binary(poses[:W2])

        def same(a, b):
            return all(np.array_equal(a[k], b[k]) for k in a if a[k] is not None)

        for _ in range(2):
            assert same(ctx.eval_unary(poses, jac_kind=0), first[0])
            assert same(ctx.eval_edge(poses[:W2]), first_e)
            assert np.array_equal(ctx.eval_unary(poses, want_jac=False)["cost"], first_c)
            assert same(ctx.eval_binary(poses[:W2]), first_b)
            assert same(ctx.eval_unary(poses, jac_kind=1), first[1])
            small = ctx.eval_unary(poses[:W2], jac_kind=0)                 # re-plans for W' (and the by-value pose path)
            for key in ("H", "g", "cost"):
                assert np.array_equal(small[key], first[0][key][:W2])
            assert ctx.eval_binary(poses[:W2], want_jac=False)["cost"] == first_b["cost"]
            assert np.array_equal(ctx.eval_edge(poses[:W2], want_jac=False)["cost"], first_e["cost"])
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------
# solve and marginalise above the by-value pose limit
# ---------------------------------------------------------------------------------------------------------------------------
def _perturbed(rng, poses, dt=0.05, dr=0.004):
    from glio_b200 import synth
    out = poses.copy()
    out[:, :3] += rng.normal(0, dt, (len(poses), 3))
    for k in range(len(poses)):
        dq = np.concatenate([[1.0], rng.normal(0, dr, 3)]); dq /= np.linalg.norm(dq)
        out[k, 3:] = synth.quat_mul(poses[k, 3:], dq)
    return out


def test_window_solve_66(oracle):
    rng = np.random.default_rng(600)
    W = 66
    truth = er.make_poses(W, rng)
    per = _unary_fixture(rng, truth, [int(rng.integers(200, 600)) for _ in range(W)], noise=0.03)
    init = _perturbed(rng, truth)
    ctx = _ctx()
    try:
        _upload(ctx, per)
        prob = oracle.WindowProblem(init, None, Q_LB, T_LB, huber_delta=1.0)
        ks = range(W)
        prob.add_unary(np.concatenate([np.full(len(per[k]["cp"]), k, np.int32) for k in ks]), np.concatenate([per[k]["cp"] for k in ks]),
                       np.concatenate([per[k]["nsd"] for k in ks]),
                       ctx.params.lidar_const * np.concatenate([per[k]["weight"] for k in ks]).astype(np.float64))
        ro = prob.solve(oracle.solver_options(), mode=0)
        rg = ctx.window_solve(init)
        assert rg["summary"].num_iterations == ro["summary"].num_iterations >= 2
        assert [i["step_is_successful"] for i in rg["iterations"]] == [i["step_is_successful"] for i in ro["iterations"]]
        assert len(rg["steps"]) == len(ro["steps"]) > 0
        for a, b in zip(rg["steps"], ro["steps"]):
            a = a.reshape(W, 6); b = b.reshape(W, 6)
            assert np.max(np.abs(a[:, :3] - b[:, :3])) <= 1e-6 and np.max(2 * np.linalg.norm(a[:, 3:] - b[:, 3:], axis=1)) <= 1e-8
    finally:
        ctx.close()


def _marg_factors(api, oracle_prob, poses, sb):
    from glio_b200 import synth
    W = len(poses)
    sw = np.concatenate([np.full(3, 20.0), np.full(3, 50.0), np.full(9, 5.0)])
    hf = api.HostFactorSet()
    args = [(0, poses[0, :3], poses[0, 3:], sb[0], sw)]
    hf.add_prior(*args[0])
    if oracle_prob is not None:
        oracle_prob.add_prior(*args[0])
    for i in range(W - 1):
        dq = synth.quat_mul(synth.quat_conj(poses[i, 3:]), poses[i + 1, 3:]); dp = synth.quat_to_R(poses[i, 3:]).T @ (poses[i + 1, :3] - poses[i, :3])
        a = (i, i + 1, dp, dq, np.zeros(3), 0.1, sw * 0.5)
        hf.add_between(*a)
        if oracle_prob is not None:
            oracle_prob.add_between(*a)
    return hf


def test_window_marginalize_65(oracle):
    """The marginalisation at W = 65 (poses uploaded to the device) against the oracle; then the race the pinned pose buffer had:
    an asynchronous marginalisation, a per-residual evaluation of KF0 at another pose while it runs, and the prior must equal
    the synchronous pass.  (The race depends on timing: this covers the sequence, it cannot reliably provoke the old failure.)"""
    from glio_b200 import api
    rng = np.random.default_rng(650)
    W = 65
    poses = er.make_poses(W, rng, spread=5.0)
    per = _unary_fixture(rng, poses, [int(rng.integers(200, 800)) for _ in range(W)])
    sb = rng.normal(0, 0.05, (W, 9))
    ctx = _ctx()
    try:
        _upload(ctx, per)
        prob = oracle.WindowProblem(poses, sb, Q_LB, T_LB, huber_delta=1.0)
        ks = range(W)
        prob.add_unary(np.concatenate([np.full(len(per[k]["cp"]), k, np.int32) for k in ks]), np.concatenate([per[k]["cp"] for k in ks]),
                       np.concatenate([per[k]["nsd"] for k in ks]),
                       ctx.params.lidar_const * np.concatenate([per[k]["weight"] for k in ks]).astype(np.float64))
        hf = _marg_factors(api, prob, poses, sb)
        om = prob.marginalize(eps=1e-8, mode=0)
        ref = ctx.window_marginalize(poses, sb, hf).arrays()
        JtJ_o = om["lin_jac"].T @ om["lin_jac"]; Jtr_o = om["lin_jac"].T @ om["lin_res"]
        assert np.max(np.abs(ref["A_info"] - JtJ_o)) <= 1e-9 * np.abs(JtJ_o).max()
        assert np.max(np.abs(ref["b_info"] - Jtr_o)) <= 1e-8 * np.abs(Jtr_o).max()
        other = poses[0].copy(); other[:3] += 1.0
        for _ in range(3):
            job = ctx.window_marginalize_async(poses, sb, hf)
            r, J = ctx.eval_unary_residuals(0, other, len(per[0]["cp"]))
            got = job.wait().arrays()
            for key in ("lin_jac", "lin_res", "A_info", "b_info", "x0_pose", "x0_sb"):
                assert np.array_equal(got[key], ref[key]), key
            R = er.unary_residuals(other, per[0]["cp"], per[0]["nsd"], per[0]["weight"], Q_LB, T_LB, ctx.params.lidar_const, 1.0)
            er.assert_within(r, R["r"], R["Mr"], "KF0 residuals during the marginalisation")
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------
# K2b: binary plane factors
# ---------------------------------------------------------------------------------------------------------------------------
def _check_binary(ctx, poses, pairs, nonvacuous=False):
    R = er.binary_blocks(poses, pairs, ctx.params.batch_score)
    d = ctx.eval_binary(poses)
    _note("binary", er.assert_within(d["Hdiag"], R["Hdiag"], R["MHdiag"], "binary Hdiag"))
    _note("binary", er.assert_within(d["g"], R["g"], R["Mg"], "binary g"))
    _note("binary", er.assert_within(d["Hoff"], R["Hoff"], R["MHoff"], "binary Hoff"))
    _note("binary", er.assert_within(d["cost"], R["cost"], R["Mcost"], "binary cost"))
    _note("binary", er.assert_within(ctx.eval_binary(poses, want_jac=False)["cost"], R["cost"], R["Mcost"], "binary cost-only"))
    if nonvacuous:
        for H, M in ((R["Hdiag"], R["MHdiag"]), (R["Hoff"], R["MHoff"])):
            for k in range(len(H)):
                if np.max(np.abs(H[k])) > 0:
                    assert er.KAPPA * er.U * np.max(M[k]) < 1e-9 * np.max(np.abs(H[k]))
    return d, R


def _binary_oracle(oracle, ctx, poses, pairs, d):
    kc, ko, cp, nc, w = [], [], [], [], []
    for cur, oth, m in pairs:
        if m is None or not len(m["cp"]):
            continue
        n = len(m["cp"]); kc.append(np.full(n, cur, np.int32)); ko.append(np.full(n, oth, np.int32))
        cp.append(m["cp"]); nc.append(m["nc"]); w.append(m["weight"])
    o = oracle.eval_binary(poses, np.concatenate(kc), np.concatenate(ko), np.concatenate(cp), np.concatenate(nc),
                           ctx.params.batch_score * np.concatenate(w).astype(np.float64), huber_delta=0.0, mode=0)
    K = len(poses)
    for k in range(K):
        Hk = o["H"][6 * k:6 * k + 6, 6 * k:6 * k + 6]
        if np.abs(Hk).max() > 0:
            assert np.max(np.abs(d["Hdiag"][k] - Hk)) <= REL * np.abs(Hk).max()
    seen = set()
    for p, (cur, oth, m) in enumerate(pairs):
        if (min(cur, oth), max(cur, oth)) in seen:
            continue             # both directions of a pair share the oracle's off-diagonal entry
        seen.add((min(cur, oth), max(cur, oth)))
        Ho = o["H"][6 * cur:6 * cur + 6, 6 * oth:6 * oth + 6]
        both = [q for q, (c2, o2, _) in enumerate(pairs) if {c2, o2} == {cur, oth}]
        got = sum(d["Hoff"][q] if pairs[q][0] == cur else d["Hoff"][q].T for q in both)
        assert np.max(np.abs(got - Ho)) <= REL * max(np.abs(Ho).max(), 1e-300)
    assert abs(d["cost"] - o["cost_total"]) <= REL * abs(o["cost_total"])


BIN_COUNTS = [0, 1, 127, 128, 129, 2048, 2049, 4097]


def test_binary_counts_and_layout(oracle):
    """Pair match counts around the 128-thread block and the 2048-residual item, both directions of a pair, spans up to 10,
    keyframes without any incidence, and declared pairs that never get matches (they contribute exactly zero)."""
    rng = np.random.default_rng(700)
    K = 24
    poses = er.make_poses(K, rng)
    layout = [(0, 1), (1, 0), (2, 12), (12, 2), (5, 6), (6, 9), (9, 19), (13, 14), (20, 23), (23, 21)]
    ctx = _ctx()
    try:
        ctx.batch_declare_pairs([4, 15], [16, 4])           # declared, never matched
        pairs = [(4, 16, None), (15, 4, None)]
        for i, (cur, oth) in enumerate(layout):
            n = BIN_COUNTS[i % len(BIN_COUNTS)]
            m = er.make_pair(rng, poses[cur], poses[oth], n)
            ctx.batch_set_pair_matches(cur, oth, m["cp"], m["nc"], m["weight"])
            pairs.append((cur, oth, m))
        assert [tuple(x) for x in zip(*ctx.batch_pair_list())] == [(c, o) for c, o, _ in pairs]
        d, R = _check_binary(ctx, poses, pairs, nonvacuous=True)
        assert not d["Hoff"][0].any() and not d["Hoff"][1].any()
        idle = [k for k in range(K) if k not in {x for c, o, m in pairs if m is not None and len(m["cp"]) for x in (c, o)}]
        assert 4 in idle and all(not d["Hdiag"][k].any() and not d["g"][k].any() for k in idle)
        _binary_oracle(oracle, ctx, poses, pairs, d)
    finally:
        ctx.close()


def test_binary_large_k_offsets_and_nonunit():
    """K = 200 keyframes at 3 and 20 km with pose quaternions of norm 0.5 / 2 in the cost (tangent blocks at unit norm)."""
    rng = np.random.default_rng(710)
    K = 200
    poses = er.make_poses(K, rng, offset=np.where(np.arange(K) % 2, 3000.0, 20000.0))
    ctx = _ctx()
    try:
        pairs = []
        for i in range(0, K - 10, 3):
            cur, oth = i, i + 1 + (i % 10)
            m = er.make_pair(rng, poses[cur], poses[oth], int(rng.integers(1, 3000)))
            ctx.batch_set_pair_matches(cur, oth, m["cp"], m["nc"], m["weight"])
            pairs.append((cur, oth, m))
        _check_binary(ctx, poses, pairs)
        nonunit = poses.copy(); nonunit[:, 3:] *= np.where(np.arange(K) % 2, 0.5, 2.0)[:, None]
        R = er.binary_blocks(nonunit, pairs, ctx.params.batch_score)
        c = ctx.eval_binary(nonunit, want_jac=False)["cost"]
        _note("binary", er.assert_within(c, R["cost"], R["Mcost"], "binary cost, non-unit q"))
    finally:
        ctx.close()


def test_declare_pairs_rejects_malformed():
    """(-1, 2) and (3, 3) are refused with GLIO_ERR_ARG and leave the pair list as it was; evaluation then runs normally."""
    from glio_b200 import api
    rng = np.random.default_rng(720)
    K = 5
    poses = er.make_poses(K, rng)
    ctx = _ctx()
    try:
        m = er.make_pair(rng, poses[0], poses[1], 900)
        ctx.batch_set_pair_matches(0, 1, m["cp"], m["nc"], m["weight"])
        before = ctx.batch_pair_list()
        for cur, oth in (([2, -1], [3, 2]), ([1, 3], [4, 3]), ([2], [-5])):
            with pytest.raises(api.GlioError):
                ctx.batch_declare_pairs(cur, oth)
            after = ctx.batch_pair_list()
            assert np.array_equal(after[0], before[0]) and np.array_equal(after[1], before[1])
        _check_binary(ctx, poses, [(0, 1, m)])
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------
# K2e: point-to-edge factors
# ---------------------------------------------------------------------------------------------------------------------------
def _check_edge(ctx, poses, per_kf, huber=1.0, nonvacuous=False):
    R = er.unary_blocks(poses, per_kf, Q_LB, T_LB, 0.0, huber, fn="edge")
    d = ctx.eval_edge(poses)
    _note("edge", er.assert_within(d["H"], R["H"], R["MH"], "edge H"))
    _note("edge", er.assert_within(d["g"], R["g"], R["Mg"], "edge g"))
    _note("edge", er.assert_within(d["cost"], R["cost"], R["Mcost"], "edge cost"))
    _note("edge", er.assert_within(ctx.eval_edge(poses, want_jac=False)["cost"], R["cost"], R["Mcost"], "edge cost-only"))
    if nonvacuous:
        # 1e-8, not 1e-9: the distance to the line is a difference of coordinates a few hundred times larger (lp - a with
        # |lp| ~ 40 m against 8 cm), so fp64 itself cannot do better; a dropped residual still moves H by ~1/n
        for k in range(len(poses)):
            if np.max(np.abs(R["H"][k])) > 0:
                assert er.KAPPA * er.U * np.max(R["MH"][k]) < 1e-8 * np.max(np.abs(R["H"][k]))
    return d, R


def test_edge_counts_windows_and_offsets(oracle):
    rng = np.random.default_rng(800)
    counts = [1, 255, 256, 257, 2047, 2048, 2049, 4097, 6000]
    W = 70
    poses = er.make_poses(W, rng)
    ctx = _ctx()
    try:
        per = [er.make_edges(rng, poses[k], counts[k % len(counts)], Q_LB, T_LB) if k % 7 else None for k in range(W)]
        for k, e in enumerate(per):
            if e is not None:
                ctx.set_edges(k, e["cp"], e["pa"], e["pb"], e["s"])
        d, R = _check_edge(ctx, poses, per, nonvacuous=True)
        ks = [k for k in range(W) if per[k] is not None]
        kf = np.concatenate([np.full(len(per[k]["cp"]), k, np.int32) for k in ks])
        cat = {key: np.concatenate([per[k][key] for k in ks]) for key in ("cp", "pa", "pb", "s")}
        o = oracle.eval_edge(poses, Q_LB, T_LB, kf, cat["cp"], cat["pa"], cat["pb"], cat["s"], huber_delta=1.0, mode=0)
        _assert_oracle(o, kf, d, W)
        # km offsets, mixed in one window
        far = er.make_poses(W, rng, offset=np.where(np.arange(W) % 2, 3000.0, 20000.0))
        per = [er.make_edges(rng, far[k], counts[k % len(counts)], Q_LB, T_LB) for k in range(W)]
        for k, e in enumerate(per):
            ctx.set_edges(k, e["cp"], e["pa"], e["pb"], e["s"])
        _check_edge(ctx, far, per)
        # non-unit pose quaternions: the cost (the Jacobian's rotation columns share the unary tangent caveat)
        nonunit = far.copy(); nonunit[:, 3:] *= np.where(np.arange(W) % 2, 0.5, 2.0)[:, None]
        R = er.unary_blocks(nonunit, per, Q_LB, T_LB, 0.0, 1.0, fn="edge")
        _note("edge", er.assert_within(ctx.eval_edge(nonunit, want_jac=False)["cost"], R["cost"], R["Mcost"], "edge cost, non-unit q"))
    finally:
        ctx.close()
