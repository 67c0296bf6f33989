"""The device IMU row against the independent reference (tests/imu_reference.py) on the edges of tests/imu_cases.py:
dl_imu_preintegrate and every predicted state bit for bit (dl_imu.cu is built with -fmad=false), the prepared factor's
information matrix bit for bit, and the fused solve's IMU normal equations (dl_nls.cu, -fmad=true) within 1e-11 of the
reference's scale."""
import numpy as np
import pytest

import imu_cases
import imu_reference as R
from helpers import pose_error, workload

pytestmark = pytest.mark.gpu
BATCHES = imu_cases.batches()
MISMATCH = imu_cases.MISMATCH


@pytest.fixture(scope="module")
def ctx():
    import dliom
    c = dliom.Context(0)
    yield c
    c.close()


def bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float64)).view(np.uint64)


def preint_fields(m):
    return {"sum_dt": [m.sum_dt], "delta_p": m.dp, "delta_q": m.dq, "delta_v": m.dv, "linearized_ba": m.ba,
            "linearized_bg": m.bg, "jacobian": np.ravel(m.J), "covariance": np.ravel(m.P)}


def device_preintegrate(ctx, noise, batch):
    return ctx.imu_preintegrate(noise, [iv for iv, _, _ in batch], np.array([np.concatenate([ba, bg]) for _, ba, bg in batch]))


@pytest.mark.parametrize("name", list(BATCHES))
def test_preintegration_is_the_reference_bit_for_bit(ctx, name):
    reason, noise, batch = BATCHES[name]
    got = device_preintegrate(ctx, noise, batch)
    equal = total = 0
    for k, (iv, ba, bg) in enumerate(batch):
        want = preint_fields(R.preintegrate(noise, ba, bg, *iv))
        for field, w in want.items():
            g = getattr(got[k], field)
            g = [g] if isinstance(g, float) else list(g)
            same = np.array_equal(bits(g), bits(np.ravel(w)))
            equal += same
            total += 1
            assert same, (name, k, field, reason)
    print(f"{name}: {equal}/{total} fields bit-equal over {len(batch)} intervals")


@pytest.mark.parametrize("name", ["bench_20", "past_pi", "spin_12", "gap_half_second", "batch_37", "long_2001"])
def test_dl_imu_predict_is_the_reference_bit_for_bit(ctx, name):
    _, noise, batch = BATCHES[name]
    got = device_preintegrate(ctx, noise, batch)
    for k, (iv, ba, bg) in enumerate(batch):
        si = imu_cases.state_i(k, ba, bg)
        assert np.array_equal(bits(ctx.imu_predict(si, got[k])), bits(R.predict(si, R.preintegrate(noise, ba, bg, *iv)))), k


# ------------------------------------------------------------------ the prepared factor and the IMU normal equations
def _x16(f, pert):
    delta = imu_cases.perturbations()[pert][1]
    if isinstance(delta, str):
        x = list(f.x16)
        x[3:7] = [-v for v in x[3:7]]
        return np.array(x)
    return np.array(R.plus(f.x16, delta, R.FP64))


def check_normal_equations(out, k, f, x, tag):
    """H within 1e-11 sqrt(H_aa H_bb); r within 1e-11 of the magnitude of the terms it is formed from; g and cost2 within
    the bounds those imply (|J|^T |W| (|r| + s) and (|r| + s)^T |W| (|r| + s), times 1e-11)."""
    r, H, g, c2 = f.normal_equations(list(x))
    J, W = np.abs(f.jacobian(list(x))), np.abs(f.W)
    s = 1 + np.abs(x).max() + np.abs(f.pi).max() + np.abs(f.vi).max() * (1 + f.m.sum_dt) + 10 * (1 + f.m.sum_dt) ** 2
    d = np.sqrt(np.abs(np.diag(H)))
    assert np.all(np.abs(out["hessian"][k] - H) <= 1e-11 * np.outer(d, d) + 1e-300), tag
    assert np.all(np.abs(out["residual"][k] - r) <= 1e-11 * s), tag
    rs = np.abs(r) + s
    assert np.all(np.abs(out["gradient"][k] - g) <= 1e-11 * (J.T @ (W @ rs))), tag
    assert abs(out["cost2"][k] - c2) <= 1e-11 * (rs @ W @ rs), tag


def factor_problems(mismatch):
    """Every submap pose x state-j placement x imu_weight, on the bench-shaped interval."""
    _, noise, batch = BATCHES["bench_20"]
    iv, ba, bg = batch[0]
    probs = []
    for si_seed, (sname, (_, pose)) in enumerate(imu_cases.SUBMAPS.items()):
        si = imu_cases.state_i(si_seed, ba + (MISMATCH[0] if mismatch else 0), bg + (MISMATCH[1] if mismatch else 0))
        for pert in imu_cases.perturbations():
            for w in imu_cases.WEIGHTS:
                probs.append((f"{sname}/{pert}/w={w}", si, pose, w, pert))
    return noise, iv, ba, bg, probs


def run_factor_cases(ctx, mismatch):
    noise, iv, ba, bg, probs = factor_problems(mismatch)
    pre = ctx.imu_preintegrate(noise, [iv], np.array([np.concatenate([ba, bg])]))[0]
    m = R.preintegrate(noise, ba, bg, *iv)
    ref = [R.Factor(si, m, pose, imu_weight=w) for _, si, pose, w, _ in probs]
    xs = [_x16(f, p[4]) for f, p in zip(ref, probs)]
    # the prepared start (x16 = NULL) and an explicit state j, in one launch each
    start = ctx.imu_factor_evaluate([p[1] for p in probs], [pre] * len(probs), [p[2] for p in probs],
                                    imu_weight=1.0)  # weight-independent fields; W is compared below per weight
    out = {}
    for w in imu_cases.WEIGHTS:
        idx = [k for k, p in enumerate(probs) if p[3] == w]
        sub = ctx.imu_factor_evaluate([probs[k][1] for k in idx], [pre] * len(idx), [probs[k][2] for k in idx], imu_weight=w,
                                      x16=[xs[k] for k in idx])
        for j, k in enumerate(idx):
            out[k] = {key: v[j] for key, v in sub.items()}
    exact = 0
    for k, (tag, si, pose, w, pert) in enumerate(probs):
        f, o = ref[k], out[k]
        assert o["ok"] == 1 and start["ok"][k] == 1, tag
        assert np.array_equal(bits(o["predicted"]), bits(f.predicted)), tag
        assert np.array_equal(bits(start["predicted"][k]), bits(f.predicted)), tag
        assert np.array_equal(bits(o["information"]), bits(f.W)), tag
        exact += 1
        check_normal_equations({key: [v] for key, v in o.items()}, 0, f, xs[k], tag)
        if pert == "start" and w == 1.0:
            check_normal_equations(start, k, f, np.array(f.x16), tag + " (prepared start)")
    print(f"{'mismatched' if mismatch else 'linearisation'} biases: {exact}/{len(probs)} factors with ok, predicted and W "
          f"bit-equal")


def test_factor_evaluate_at_the_linearisation_biases(ctx):
    run_factor_cases(ctx, mismatch=False)


def test_factor_evaluate_with_mismatched_biases_applies_the_bias_correction(ctx):
    """State i's biases 0.05 m/s^2 and 5e-3 rad/s away from the pre-integration's: the device residual must carry the
    first-order correction of integration_base.h:283-290."""
    run_factor_cases(ctx, mismatch=True)


def test_factor_evaluate_rejects_a_singular_covariance(ctx):
    for name in ("zero_random_walk", "one_step", "one_sample", "empty_first"):
        _, noise, batch = BATCHES[name]
        iv, ba, bg = batch[0]
        pre = device_preintegrate(ctx, noise, [batch[0]])[0]
        good = device_preintegrate(ctx, BATCHES["bench_20"][1], BATCHES["bench_20"][2])[0]
        si = imu_cases.state_i(0, ba, bg)
        gi = imu_cases.state_i(1, *BATCHES["bench_20"][2][0][1:])
        out = ctx.imu_factor_evaluate([gi, si, gi], [good, pre, good], [imu_cases.SUBMAPS["yaw90"][1]] * 3)
        assert out["ok"].tolist() == [1, 0, 1], name
        assert not out["information"][1].any() and not out["hessian"][1].any() and out["cost2"][1] == 0
        assert np.array_equal(bits(out["information"][0]), bits(out["information"][2]))
        assert R.information(R.preintegrate(noise, ba, bg, *iv).P, 1.0) is None


# ------------------------------------------------------------------ the front end
def _front_end(w, seed):
    """The workload's scans with raw 200 Hz samples along their trajectory and states i carrying distinct biases."""
    import imu_synth
    intervals, states_i = [], []
    for s in range(len(w["scans"])):
        t1 = w["times"][s]
        intervals.append(imu_synth.samples(t1 - 0.1, t1, noise=(3.99e-2, 1.56e-2), seed=seed + s))
        ba, bg = imu_cases.biases(seed + s)
        states_i.append(imu_synth.state(t1 - 0.1, ba=ba, bg=bg))
    return intervals, states_i


NOISE = list(R.KAIST_NOISE)


@pytest.fixture(scope="module")
def scene(ctx):
    import dliom
    w = workload()
    return w, dliom.Grid.from_oracle(ctx, w["hi"]), dliom.Grid.from_oracle(ctx, w["lo"]), dliom.FrontendOptions.from_oracle(w["opts"])


def test_front_end_predictions_read_biases_at_stride_16(ctx, scene):
    """dl_frontend_match_batch_imu_samples reads state i's biases from the 16-double nav states; its predictions equal the
    reference's, bit for bit, and its estimates equal those of the host-prepared chain fed the same predictions and
    dl_imu_preintegrate's pre-integrations (the two factor builders share every operation)."""
    import dliom
    w, hi, lo, fo = scene
    intervals, states_i = _front_end(w, 50)
    imu = dliom.ImuSamples(NOISE, intervals, states_i, imu_weight=0.7)
    res, states, predicted = ctx.frontend_match_batch_imu_samples(fo, w["scans"], w["origin"], imu, w["submap_pose"], hi, lo)
    preints = []
    for s, (iv, si) in enumerate(zip(intervals, states_i)):
        m = R.preintegrate(NOISE, si[10:13], si[13:16], *iv)
        assert np.array_equal(bits(predicted[s]), bits(R.predict(si, m))), s
        preints.append(ctx.imu_preintegrate(NOISE, [iv], np.array([si[10:16]]))[0])
        assert res[s].ok == 1
    res_h, states_h = ctx.frontend_match_batch_imu(fo, w["scans"], w["origin"], states_i, predicted, preints, w["submap_pose"],
                                                   hi, lo, imu_weight=0.7)
    for s in range(len(states_i)):
        assert res_h[s].summary.num_iterations == res[s].summary.num_iterations, s
        assert np.array_equal(states_h[s], states[s]), (s, states_h[s] - states[s])


def test_front_end_marks_a_singular_interval_and_leaves_the_others(ctx, scene):
    """A one-sample interval has P = 0: ok = -2 for its scan, every other scan's state and result byte-identical."""
    import dliom
    w, hi, lo, fo = scene
    intervals, states_i = _front_end(w, 60)
    full = dliom.ImuSamples(NOISE, intervals, states_i, imu_weight=0.7)
    res, states, _ = ctx.frontend_match_batch_imu_samples(fo, w["scans"], w["origin"], full, w["submap_pose"], hi, lo)
    holed = list(intervals)
    holed[2] = tuple(a[:1] for a in intervals[2])
    imu = dliom.ImuSamples(NOISE, holed, states_i, imu_weight=0.7)
    res2, states2, _ = ctx.frontend_match_batch_imu_samples(fo, w["scans"], w["origin"], imu, w["submap_pose"], hi, lo)
    assert res2[2].ok == -2
    for s in range(len(states_i)):
        if s == 2:
            continue
        assert res2[s].ok == 1 and bytes(res2[s]) == bytes(res[s]) and np.array_equal(bits(states2[s]), bits(states[s])), s


# ------------------------------------------------------------------ the fused solve at mismatched biases
def test_fused_solve_with_mismatched_biases_matches_the_oracle(ctx, orc, scene):
    """dl_fused_match_batch with pre-integrations linearised at other biases than state i's: the oracle applies the
    bias correction, so must the device (tolerances of test_gpu_imu.py)."""
    import imu_synth
    w, hi, lo, _ = scene
    for s in range(len(w["scans"])):
        t1 = w["times"][s]
        dt, acc, gyr = imu_synth.samples(t1 - 0.1, t1, noise=(3.99e-2, 1.56e-2), seed=70 + s)
        lin_ba, lin_bg = np.zeros(3), np.zeros(3)
        si = imu_synth.state(t1 - 0.1, ba=MISMATCH[0], bg=MISMATCH[1])
        m = orc.imu_preintegrate(NOISE, lin_ba, lin_bg, dt, acc, gyr)
        pred = orc.imu_predict(si, m)
        ing = orc.ingest_scan(w["opts"], w["scans"][s], w["origin"], si[:7], pred[:7])
        pts = ing["returns_tracking"]
        hk, _ = orc.adaptive_voxel_filter(pts, 2.0, 150, 15.0)
        lk, _ = orc.adaptive_voxel_filter(pts, 4.0, 200, 60.0)
        init = pred.copy()
        init[:3] += [0.03, -0.02, 0.01]
        dev_m = ctx.imu_preintegrate(NOISE, [(dt, acc, gyr)], np.zeros((1, 6)))[0]
        for tw, rw, iw in ((0.0, 0.0, 1.0), (5.0, 4e2, 0.5)):
            want, ws = orc.fused_match([pts[hk], pts[lk]], [w["hi"], w["lo"]], [1.0, 6.0], tw, rw, init[:3], si, init, m,
                                       imu_weight=iw)
            got, gs = ctx.fused_match_batch([[pts[hk], pts[lk]]], [[hi, lo]], [1.0, 6.0], tw, rw, [w["submap_pose"]], [si],
                                            [init], [dev_m], imu_weight=iw)
            dtn, drn = pose_error(got[0][:7], want[:7])
            assert dtn < 1e-7 and drn < 1e-8, (s, dtn, drn)
            assert np.allclose(got[0][7:], want[7:], atol=1e-7)
            assert gs[0]["num_iterations"] == ws["num_iterations"]
