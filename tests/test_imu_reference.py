"""CPU checks of the IMU reference (tests/imu_reference.py): known physics, its fp64 error against 50-digit mpmath, its
derivatives, and the C++ oracle (oracle/orc_imu.h) against it."""
import math

import numpy as np
import pytest

import imu_cases
import imu_reference as R

EPS = np.finfo(np.float64).eps
BATCHES = imu_cases.batches()


def bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float64)).view(np.uint64)


def test_case_generators_hit_their_edges():
    b = BATCHES
    m = R.preintegrate(b["past_pi"][1], *_args(b["past_pi"][2][0]))
    assert m.dq[0] < 0                                  # passed pi
    m = R.preintegrate(b["one_sample"][1], *_args(b["one_sample"][2][0]))
    assert m.sum_dt == 0 and np.array_equal(m.J, np.eye(15)) and not m.P.any()
    m = R.preintegrate(b["short_5ms"][1], *_args(b["short_5ms"][2][0]))
    assert np.linalg.cond(m.P) >= 1e10
    m = R.preintegrate(b["zero_random_walk"][1], *_args(b["zero_random_walk"][2][0]))
    assert R.information(m.P, 1.0) is None
    m = R.preintegrate(b["one_step"][1], *_args(b["one_step"][2][0]))
    assert R.information(m.P, 1.0) is None
    iv, _, bg = b["bg_equals_omega"][2][0]
    un_gyr = 0.5 * (iv[2][:-1] + iv[2][1:]) - bg
    assert np.abs(un_gyr).max() < 0.05 * np.abs(iv[2]).max()
    assert np.abs(b["saturated_16g"][2][0][0][1]).max() == imu_cases.G16
    assert [len(x[0][0]) for x in b["empty_middle"][2]] == [20, 0, 20]
    assert len(b["batch_37"][2]) == 37 and {0, 1, 150} <= {len(x[0][0]) for x in b["batch_37"][2]}


def _args(entry):
    iv, ba, bg = entry
    return ba, bg, iv[0], iv[1], iv[2]


# ------------------------------------------------------------------ physics
def test_constant_rate_gives_the_closed_form_rotation():
    w = np.array([0.4, -1.1, 2.3])
    dt, n = 0.005, 400
    m = R.preintegrate(R.KAIST_NOISE, (0, 0, 0), (0, 0, 0), np.full(n + 1, dt), np.zeros((n + 1, 3)), np.tile(w, (n + 1, 1)))
    phi = math.atan(np.linalg.norm(w) * dt / 2)
    want = np.concatenate([[math.cos(n * phi)], math.sin(n * phi) * w / np.linalg.norm(w)])
    assert np.abs(np.array(m.dq) - want).max() <= 8 * n * EPS
    assert m.dp == (0.0, 0.0, 0.0) and m.dv == (0.0, 0.0, 0.0)


def test_constant_acceleration_without_rotation():
    a = np.array([0.7, -0.3, 9.8])
    dt, n = 0.005, 400
    m = R.preintegrate(R.KAIST_NOISE, (0, 0, 0), (0, 0, 0), np.full(n + 1, dt), np.tile(a, (n + 1, 1)), np.zeros((n + 1, 3)))
    T = m.sum_dt
    assert abs(T - n * dt) <= n * EPS * T
    assert np.abs(np.array(m.dp) - 0.5 * a * T * T).max() <= 4 * n * EPS * np.abs(0.5 * a * T * T).max()
    assert np.abs(np.array(m.dv) - a * T).max() <= 4 * n * EPS * np.abs(a * T).max()
    assert m.dq == (1.0, 0.0, 0.0, 0.0)


# ------------------------------------------------------------------ precision against 50 digits
PRECISION = ["two_samples", "bench_20", "jitter30", "zero_dt", "tiny_dt", "gap_half_second", "spin_12", "ba_half",
             "saturated_16g", "short_5ms"]


@pytest.mark.parametrize("name", PRECISION)
def test_fp64_reference_error_grows_at_most_linearly(name):
    """|fp64 - exact| <= 64 (n + 1) eps max|x| for every delta, sum_dt, J and P (n = number of steps)."""
    noise, batch = BATCHES[name][1], BATCHES[name][2]
    for entry in batch:
        m = R.preintegrate(noise, *_args(entry))
        e = R.preintegrate(noise, *_args(entry), A=R.Exact())
        n = max(len(entry[0][0]) - 1, 0)
        bound = 64 * (n + 1) * EPS
        for got, want in ((m.dp, e.dp), (m.dv, e.dv), (m.dq, e.dq), ((m.sum_dt,), (e.sum_dt,)), (m.J, e.J), (m.P, e.P)):
            want = np.array(want, dtype=object).ravel()
            err = max(abs(float(w - g)) for g, w in zip(np.ravel(got), want))
            scale = max(abs(float(w)) for w in want)
            assert err <= bound * scale, (name, err, scale)


@pytest.mark.parametrize("name", ["bench_20", "short_5ms", "long_2001", "spin_12", "jitter30"])
@pytest.mark.parametrize("weight", imu_cases.WEIGHTS)
def test_information_times_covariance_is_weight_squared_identity(name, weight):
    """W Sigma = w² I within 64 cond(Sigma) eps, with the product taken exactly."""
    noise, entry = BATCHES[name][1], BATCHES[name][2][0]
    m = R.preintegrate(noise, *_args(entry))
    W = R.information(m.P, weight)
    E = R.Exact()
    S = [[E.num(v) for v in row] for row in m.P]
    cond = np.linalg.cond(m.P)
    worst = 0.0
    for a in range(15):
        for b in range(15):
            s = sum((E.num(W[a, k]) * S[k][b] for k in range(15)), E.num(0))
            worst = max(worst, abs(float(s - (weight * weight if a == b else 0))))
    assert worst <= 64 * cond * EPS * weight * weight, (worst, cond)


# ------------------------------------------------------------------ derivatives
FACTORS = [(s, p) for s in imu_cases.SUBMAPS for p in imu_cases.perturbations()]


def _factor_inputs(seed, mismatch):
    noise, entry = BATCHES["bench_20"][1], BATCHES["bench_20"][2][0]
    iv, ba, bg = entry
    si = imu_cases.state_i(seed, ba + (imu_cases.MISMATCH[0] if mismatch else 0), bg + (imu_cases.MISMATCH[1] if mismatch else 0))
    return noise, iv, ba, bg, si


def state_j(f, pert, A=R.FP64):
    delta = imu_cases.perturbations()[pert][1]
    if isinstance(delta, str):
        x = list(f.x16)
        x[3:7] = [-v for v in x[3:7]]
        return x
    return R.plus(f.x16, delta, A)


@pytest.mark.parametrize("submap,pert", FACTORS)
def test_residual_jacobian_matches_mpmath_central_differences(submap, pert):
    noise, iv, ba, bg, si = _factor_inputs(3, True)
    pose = imu_cases.SUBMAPS[submap][1]
    m = R.preintegrate(noise, ba, bg, *iv)
    f = R.Factor(si, m, pose)
    x = state_j(f, pert)
    J = f.jacobian(x)
    E = R.Exact()
    me = R.preintegrate(noise, ba, bg, *iv, A=E)
    fe = R.Factor(si, me, pose)
    h = E.ctx.mpf("1e-20")
    for c in range(15):
        d = [E.num(0)] * 15
        d[c] = h
        rp = fe.residual(R.plus(x, d, E))
        d[c] = -h
        rm = fe.residual(R.plus(x, d, E))
        col = [float((a - b) / (2 * h)) for a, b in zip(rp, rm)]
        assert np.abs(np.array(col) - J[:, c]).max() <= 1e-8, (c, col, J[:, c])


def test_bias_blocks_of_the_jacobian_are_first_order_reintegration():
    noise, entry = BATCHES["bench_20"][1], BATCHES["bench_20"][2][0]
    iv, ba, bg = entry
    m = R.preintegrate(noise, ba, bg, *iv)
    for dba, dbg in (((1e-4, -2e-4, 1e-4), (0, 0, 0)), ((0, 0, 0), (1e-5, 2e-5, -1e-5))):
        dba, dbg = np.array(dba, float), np.array(dbg, float)
        m2 = R.preintegrate(noise, ba + dba, bg + dbg, *iv)
        db = np.concatenate([dba, dbg])
        e = R.qmul(R.conj(m.dq), m2.dq)
        got = np.concatenate([np.subtract(m2.dp, m.dp), 2 * np.array(e[1:]), np.subtract(m2.dv, m.dv)])
        lin = m.J[0:9, 9:15] @ db
        assert np.abs(got - lin).max() <= 1e-3 * np.abs(lin).max() + 1e-14, (got, lin)


def test_bias_correction_moves_the_residual_by_the_bias_blocks():
    """The corrected residual at mismatched biases equals, to first order, the residual of a re-integration at state i's
    biases (what the correction stands in for)."""
    noise, iv, ba, bg, si = _factor_inputs(4, True)
    pose = imu_cases.SUBMAPS["yaw90"][1]
    f = R.Factor(si, R.preintegrate(noise, ba, bg, *iv), pose)
    g = R.Factor(si, R.preintegrate(noise, si[10:13], si[13:16], *iv), pose)
    x = R.plus(f.x16, imu_cases.perturbations()["moved"][1], R.FP64)
    raw = R.Factor(si, R.preintegrate(noise, ba, bg, *iv), pose)
    raw.dp, raw.dv, raw.dq_inv = raw.m.dp, raw.m.dv, R.conj(raw.m.dq)
    rf, rg, rr = (np.array(h.residual(x)) for h in (f, g, raw))
    assert np.abs(rf - rg).max() < 0.01 * np.abs(rr - rg).max()
    assert np.abs(rr - rg)[:9].max() > 1e-5


# ------------------------------------------------------------------ the oracle against the reference
ORACLE = list(BATCHES)


@pytest.mark.parametrize("name", ORACLE)
def test_oracle_preintegration_and_prediction_equal_the_reference(orc, name):
    """orc_imu.h evaluates every field in the same order as the reference: sum_dt, delta_p, delta_q, delta_v, jacobian,
    covariance and imu_predict's state are compared bit for bit."""
    noise, batch = BATCHES[name][1], BATCHES[name][2]
    for k, (iv, ba, bg) in enumerate(batch):
        m = R.preintegrate(noise, ba, bg, *iv)
        o = orc.imu_preintegrate(noise, ba, bg, *iv)
        for got, want in ((o.sum_dt, m.sum_dt), (o.delta_p, m.dp), (o.delta_q, m.dq), (o.delta_v, m.dv),
                          (o.jacobian, m.J.ravel()), (o.covariance, m.P.ravel())):
            assert np.array_equal(bits(list(got) if not isinstance(got, float) else [got]), bits(np.ravel(want))), (name, k)
        si = imu_cases.state_i(k, ba, bg)
        assert np.array_equal(bits(orc.imu_predict(si, o)), bits(R.predict(si, m))), (name, k)


@pytest.mark.parametrize("mismatch", [False, True])
@pytest.mark.parametrize("pert", list(imu_cases.perturbations()))
def test_oracle_residual_equals_the_reference(orc, mismatch, pert):
    """orc.imu_residual works in the local frame; the reference composes with the identity submap pose, which re-normalises
    q_i: compared to 1e-13 relative (of the largest term) instead of bit for bit."""
    noise, iv, ba, bg, si = _factor_inputs(5, mismatch)
    m = R.preintegrate(noise, ba, bg, *iv)
    f = R.Factor(si, m, imu_cases.SUBMAPS["identity"][1])
    x = np.array(state_j(f, pert))
    o = orc.imu_preintegrate(noise, ba, bg, *iv)
    r, J = orc.imu_residual(si, x, o)
    scale = 1 + np.abs(x).max() + np.abs(si).max() * (1 + m.sum_dt)
    assert np.abs(r - np.array(f.residual(x))).max() <= 1e-13 * scale
    assert np.abs(J - f.jacobian(x)).max() <= 1e-13
