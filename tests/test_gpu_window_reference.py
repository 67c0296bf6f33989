"""The device window update (csrc/dl_window.cu) against the independent 50-digit reference (tests/window_reference.py) on the
edges of tests/window_cases.py: the factors alone at chosen points (dl_window_evaluate), whole solves, solves stopped by the
iteration limit, a chain that carries its own information on each side, batches against single calls and failures.
Tolerances come from quantities the reference computes, never from the device's output; each is printed on failure."""
import numpy as np
import pytest

import imu_reference as ir
import window_cases as wc
import window_reference as wr
from helpers import pose_error

pytestmark = pytest.mark.gpu
EPS = np.finfo(float).eps
EXACT = ir.Exact()
CASES = wc.cases()


@pytest.fixture(scope="module")
def ctx():
    import dliom
    c = dliom.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def reference():
    return {name: wr.solve(p, EXACT) for name, (_, p) in CASES.items()}


def _pre(p):
    import dliom
    return wc.preint_struct(p["pre"], dliom.Preintegration)


def run(ctx, ps, states_i_out=True):
    """One dl_window_optimize_batch over the problems ps (all with the options of ps[0])."""
    p0 = ps[0]
    init = None if p0["initial_j"] is None else [p["initial_j"] for p in ps]
    return ctx.window_optimize_batch([p["mean_i"] for p in ps], [p["prior"] for p in ps], [_pre(p) for p in ps],
                                     [p["matched"] for p in ps], gravity=p0["G"], max_iter=p0["max_iter"], initial_j=init,
                                     states_i_out=states_i_out, **wc.options(p0))


def evaluate(ctx, p, xi, xj):
    out = ctx.window_evaluate([p["mean_i"]], [p["prior"]], [_pre(p)], [p["matched"]], [xi], [xj], gravity=p["G"], **wc.options(p))
    return {k: v[0] for k, v in out.items()}


# ------------------------------------------------------------------ the factors at chosen points
def _rotated(q, angle, axis):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    return np.array(ir.qmul(tuple(np.concatenate([[np.cos(angle / 2)], np.sin(angle / 2) * a])), tuple(q)))


def _points():
    """name -> (problem, x_i, x_j). The prior rotation error d = q_i mean^-1 is a half angle: |v| = sin(angle / 2)."""
    out = {}
    for pname in ("bias_offset", "gf_tilted", "gf_gx_above"):
        p = CASES[pname][1]
        xj0 = np.array(ir.predict(p["mean_i"], p["pre"]), float)
        xj0[:3] += [0.01, -0.02, 0.005]
        xj0[3:7] = _rotated(xj0[3:7], 0.01, (1, 2, 3))
        xi0 = p["mean_i"].copy()
        xi0[:3] += [0.003, -0.002, 0.001]
        xi0[7:16] += np.linspace(-1e-3, 1e-3, 9)                    # biases moved: the bias correction depends on x_i
        for tag, angle in (("1e-9", 2e-9), ("1e-7", 2e-7), ("below_1e-8", 2 * 0.99e-8), ("above_1e-8", 2 * 1.01e-8),
                           ("90deg", np.pi / 2)):
            xi = xi0.copy()
            xi[3:7] = _rotated(p["mean_i"][3:7], angle, (0.3, -0.5, 0.8))
            out[f"{pname}-prior_{tag}"] = (p, xi, xj0)
        xi = xi0.copy()
        xi[3:7] = -_rotated(p["mean_i"][3:7], 0.2, (1, 0, 0))        # q_i mean^-1 has w < 0
        out[f"{pname}-prior_w_negative"] = (p, xi, xj0)
        xj = xj0.copy()
        xj[3:7] = -xj0[3:7]                                          # the pose prior's flip
        out[f"{pname}-pose_flip"] = (p, xi0, xj)
        xj = xj0.copy()
        xj[3:7] = _rotated(p["matched"][3:7], np.pi / 2, (0, 1, 0))  # 90 deg pose and gravity errors
        out[f"{pname}-pose_90deg"] = (p, xi0, xj)
    return out


POINTS = _points()


@pytest.mark.parametrize("name", sorted(POINTS))
def test_factors_at_chosen_points(ctx, name):
    p, xi, xj = POINTS[name]
    d = evaluate(ctx, p, xi, xj)
    assert d["ok"] == 1
    rr, Jr, Wr = (ir.to_float(a) for a in wr.evaluate(p, xi, xj, EXACT))
    scale = wr.row_scales(p, xi, xj)
    tol = 64 * EPS * scale
    rows = slice(0, 36)
    err_r = np.abs(d["residual"][rows] - rr[rows]) / tol[rows]
    assert err_r.max() <= 1, f"{name}: residual row {err_r.argmax()} off by {err_r.max():.2f} x 64 eps x its scale {tol[err_r.argmax()]:.3e}"
    err_J = (np.abs(d["jacobian"][rows] - Jr[rows]) / tol[rows, None]).max(1)
    assert err_J.max() <= 1, f"{name}: Jacobian row {err_J.argmax()} off by {err_J.max():.2f} x 64 eps x its scale"
    # gravity rows: the tangent bases differ (Unit3's rule vs the device's), so compare what no basis changes: [r J]^T [r J]
    Md, Mr = np.column_stack([d["residual"][36:], d["jacobian"][36:]]), np.column_stack([rr[36:], Jr[36:]])
    gram_tol = 64 * EPS * 4
    assert np.abs(Md.T @ Md - Mr.T @ Mr).max() <= gram_tol, f"{name}: gravity rows' Gram matrix off, tolerance {gram_tol:.2e}"
    # weight: the prior block is copied; the IMU block within 32 eps kappa(Sigma) |Sigma^-1| w^2; the diagonal tail to rounding
    assert np.array_equal(d["weight"][:15, :15], p["prior"])
    Wi = Wr[15:30, 15:30]
    wtol = 32 * EPS * wr._cond(p["pre"].P) * np.abs(Wi).max()
    assert np.abs(d["weight"][15:30, 15:30] - Wi).max() <= wtol, f"{name}: IMU weight block, tolerance {wtol:.3e}"
    assert np.allclose(d["weight"][30:, 30:], Wr[30:, 30:], rtol=4 * EPS, atol=0)
    off = d["weight"].copy()
    off[:15, :15] = off[15:30, 15:30] = 0
    off[30:, 30:] -= np.diag(np.diag(off[30:, 30:]))
    assert not off.any()


def test_evaluate_refuses_a_singular_covariance(ctx):
    p = CASES["one_sample"][1]
    d = evaluate(ctx, p, p["mean_i"], np.array(ir.predict(p["mean_i"], p["pre"]), float))
    assert d["ok"] == 0 and not d["residual"].any() and not d["jacobian"].any() and not d["weight"].any()


# ------------------------------------------------------------------ whole solves
def _state_tolerances(name, ref, dev_i, dev_j):
    delta = np.concatenate([wr.minus(dev_i, ref["xi"]), wr.minus(dev_j, ref["xj"])])
    maha = float(np.sqrt(max(delta @ ref["H"] @ delta, 0.0)))
    assert maha <= 1e-6, f"{name}: state difference {maha:.3e} in the metric of the reference H, tolerance 1e-6"
    for a, b in ((dev_j, ref["xj"]), (dev_i, ref["xi"])):
        dt, dr = pose_error(a[:7], b[:7])
        assert dt < 1e-7 and dr < 1e-7 and np.abs(a[7:] - b[7:]).max() < 1e-7, f"{name}: states differ by more than 1e-7"


def _information_tolerance(name, ref, info):
    """Scaled entries |dS_ab| / sqrt(S_aa S_bb) of S = H_jj - H_ji H_ii^-1 H_ij: the solve with H_ii loses kappa(H_ii) and the
    subtraction cancels max_a H_jj,aa / S_aa (the bias rows, where the random walk ties x_j to x_i), so the bound is
    min(1e-4, 64 eps kappa(H_ii) max_a H_jj,aa / S_aa); 1e-4 is what tests/test_gpu_window.py requires against the oracle."""
    R = ref["information"]
    cancel = (np.diag(ref["H"])[15:] / np.diag(R)).max()
    bound = min(1e-4, max(1e-9, 64 * EPS * ref["kappa_Hii"] * cancel))
    scale = np.sqrt(np.outer(np.diag(R), np.diag(R)))
    err = (np.abs(info - R) / scale).max()
    assert err <= bound, (f"{name}: scaled information off by {err:.3e}, bound {bound:.3e} (kappa(H_ii) {ref['kappa_Hii']:.3e}, "
                          f"cancellation {cancel:.3e})")


@pytest.mark.parametrize("name", sorted(CASES))
def test_solve_matches_reference(ctx, reference, name):
    p, ref = CASES[name][1], reference[name]
    gi, gj, ginfo, gs = run(ctx, [p])
    s = gs[0]
    assert s["termination"] == ref["termination"], f"{name}: termination {s['termination']}, reference {ref['termination']}"
    if ref["termination"] == 2:
        assert not gj[0].any() and not ginfo[0].any()
        return
    margin = min([abs(np.log10(x) + 10) for x in ref["steps"]] + [9.0])
    assert margin >= 0.5, f"{name}: a reference step is within half a decade of 1e-10 ({ref['steps']})"
    extra = s["num_iterations"] - ref["iterations"]
    assert extra == 0 or (p.get("fp64_step_floor") and extra == 1), \
        f"{name}: {s['num_iterations']} iterations, reference {ref['iterations']} (steps {ref['steps']})"
    assert s["num_evaluations"] == s["num_iterations"] + 1
    for k in ("initial_cost", "final_cost"):
        assert abs(s[k] - ref[k]) <= 1e-9 * max(abs(ref[k]), 1e-12), f"{name}: {k} {s[k]!r} vs {ref[k]!r}, tolerance 1e-9 relative"
    _state_tolerances(name, ref, gi[0], gj[0])
    _information_tolerance(name, ref, ginfo[0])


def test_chain_carries_its_own_information(ctx):
    """Ten windows in a row: each side's estimate and information are its own next prior."""
    p0 = CASES["bias_offset"][1]
    truth = p0["mean_i"].copy()
    md = mr = p0["mean_i"].copy()
    idv = ir_ = p0["prior"].copy()
    for k in range(10):
        pre = wc.interval(21, 100 + k)
        truth = np.array(ir.predict(truth, pre), float)
        z = truth[:7].copy()
        z[:3] += 0.01 * np.array([np.sin(k), np.cos(k), 0.3])
        pd, pr = wr.problem(md, idv, pre, z), wr.problem(mr, ir_, pre, z)
        ref = wr.solve(pr, EXACT)
        gi, gj, ginfo, gs = run(ctx, [pd])
        assert gs[0]["termination"] == ref["termination"] == 0
        dt, dr = pose_error(gj[0][:7], ref["xj"][:7])
        assert dt < 1e-6 and dr < 1e-6 and np.abs(gj[0][7:] - ref["xj"][7:]).max() < 1e-6, f"step {k}"
        md, idv, mr, ir_ = gj[0], ginfo[0], ref["xj"], ref["information"]
        scale = np.sqrt(np.outer(np.diag(ir_), np.diag(ir_)))
        assert (np.abs(idv - ir_) / scale).max() < 1e-4, f"step {k}"
    assert np.linalg.eigvalsh(0.5 * (idv + idv.T)).min() > 0


# ------------------------------------------------------------------ batches and failures
def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a[:3], b[:3])) and a[3] == b[3]


@pytest.mark.parametrize("count", [1, 2, 3, 64, 257, 1000])
def test_batch_members_equal_single_calls(ctx, count):
    ps = wc.batch(count, count)
    whole = run(ctx, ps)
    assert all(s["termination"] == 0 for s in whole[3])
    members = range(count) if count <= 257 else list(range(0, count, 37)) + [count - 1]
    for k in members:
        single = run(ctx, [ps[k]])
        assert _same([a[k:k + 1] for a in whole[:3]] + [whole[3][k:k + 1]], single), f"member {k} of {count}"
    if count == 257:
        no_i = run(ctx, ps, states_i_out=False)
        assert no_i[0] is None and np.array_equal(no_i[1], whole[1]) and np.array_equal(no_i[2], whole[2]) and no_i[3] == whole[3]


@pytest.mark.parametrize("bad", [(0,), (1,), (4,), (0, 1, 4)])
def test_failing_members_leave_neighbours_alone(ctx, bad):
    """Members with a negated prior fail (termination 2) with zeroed outputs; member 1 shares member 0's block."""
    ps = wc.batch(5, 7)
    good = run(ctx, ps)
    mixed = [wc._with(p, prior=-p["prior"]) if k in bad else p for k, p in enumerate(ps)]
    out = run(ctx, mixed)
    for k in range(5):
        if k in bad:
            assert out[3][k]["termination"] == 2 and not out[1][k].any() and not out[2][k].any()
        else:
            assert np.array_equal(out[0][k], good[0][k]) and np.array_equal(out[1][k], good[1][k])
            assert np.array_equal(out[2][k], good[2][k]) and out[3][k] == good[3][k]


@pytest.mark.parametrize("field", ["gravity_direction", "body_reference_direction"])
@pytest.mark.parametrize("value", [(0.0, 0.0, 0.0), (np.nan, 0.0, 1.0), (np.inf, 0.0, 0.0)])
def test_directions_must_be_finite_and_non_zero(ctx, field, value):
    import dliom
    p = CASES["gf_tilted"][1]
    gf = list(p["gravity_factor"])
    gf[1 if field == "gravity_direction" else 2] = value
    q = wc._with(p, gravity_factor=tuple(gf))
    with pytest.raises(dliom.DlError) as e:
        run(ctx, [q])
    assert e.value.status == -2
    with pytest.raises(dliom.DlError) as e:
        evaluate(ctx, q, p["mean_i"], p["mean_i"])
    assert e.value.status == -2
