"""The window update's independent reference (tests/window_reference.py) on the edges of tests/window_cases.py, without a GPU:
the 50-digit run against an fp64 run of the same reference, against the C++ oracle (oracle/orc_window.h), and the properties
any correct lag-one smoother has. The device is compared to the same reference in tests/test_gpu_window_reference.py."""
import numpy as np
import pytest

import imu_reference as ir
import window_cases as wc
import window_reference as wr

EXACT = ir.Exact()
CASES = wc.cases()


@pytest.fixture(scope="module")
def exact():
    return {name: wr.solve(p, EXACT) for name, (_, p) in CASES.items()}


def _oracle(orc, p):
    return orc.window_optimize(p["mean_i"], p["prior"], wc.preint_struct(p["pre"], orc.Preintegration), p["matched"],
                               G=np.array(p["G"]), max_iter=p["max_iter"], initial_j=p["initial_j"], **wc.options(p))


def _close(a, b, tol):
    return np.abs(np.concatenate([wr.minus(a["xi"], b["xi"]), wr.minus(a["xj"], b["xj"])])).max() <= tol


@pytest.mark.parametrize("name", sorted(CASES))
def test_steps_keep_a_margin_from_the_threshold(exact, name):
    """Iteration counts can only be required to match when no step norm is near the 1e-10 convergence threshold."""
    steps = exact[name]["steps"]
    assert all(abs(np.log10(s) + 10) >= 0.5 for s in steps), f"{name}: {steps}"


@pytest.mark.parametrize("name", ["nominal", "bias_offset", "spin_past_pi", "far_iter1", "gf_gx_below", "prior_negated"])
def test_exact_matches_fp64(exact, name):
    """fp64 with h = 6e-6 differences: Jacobians to ~1e-10 relative, so states to 1e-9 times the path length (a step stopped by
    the iteration limit carries the Jacobian's error) and the information to 1e-6."""
    e, f = exact[name], wr.solve(CASES[name][1], ir.FP64)
    assert f["termination"] == e["termination"]
    if e["termination"] == 2:
        return
    assert f["iterations"] == e["iterations"] and _close(f, e, 1e-9 * max(1.0, sum(e["steps"])))
    assert abs(f["final_cost"] - e["final_cost"]) <= 1e-9 * e["final_cost"]
    assert np.abs(f["information"] - e["information"]).max() <= 1e-6 * np.abs(e["information"]).max()


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_matches_oracle(orc, exact, name):
    """The oracle differentiates in fp64 with h = 1e-6 (Jacobians to ~1e-10 relative): its iteration counts may differ where the
    convergence is slow, its estimate may not by more than 1e-8, its information by more than 1e-5 of the largest entry."""
    e, p = exact[name], CASES[name][1]
    if e["termination"] == 2:
        with pytest.raises(RuntimeError):
            _oracle(orc, p)
        return
    xi, xj, info, s = _oracle(orc, p)
    assert _close({"xi": xi, "xj": xj}, e, 1e-8 * max(1.0, sum(e["steps"]))), name
    assert abs(s["final_cost"] - e["final_cost"]) <= 1e-8 * e["final_cost"]
    assert abs(s["initial_cost"] - e["initial_cost"]) <= 1e-12 * e["initial_cost"]
    assert np.abs(info - e["information"]).max() <= 1e-5 * np.abs(e["information"]).max()


def test_zero_step_at_the_optimum(exact):
    p, e = CASES["nominal"][1], exact["nominal"]
    r, J, W = wr.evaluate(p, e["xi"], e["xj"], EXACT)
    H, g, _ = wr.normal_equations(W, J, r, EXACT)
    d = wr.cholesky_solve(H, -g, EXACT)
    assert float(EXACT.sqrt(sum(v * v for v in d))) < 1e-12


@pytest.mark.parametrize("name", ["nominal", "short_interval", "prior_wide", "gf_tilted"])
def test_information_is_the_marginal(exact, name):
    """The Schur complement is the inverse of the jj block of H^-1 (50 digits), symmetric and positive definite."""
    H, info = exact[name]["exact"]["H"], exact[name]["exact"]["info"]
    Hinv = wr.cholesky_solve(H, EXACT.eye(30), EXACT)
    inv = wr.cholesky_solve(Hinv[15:, 15:].copy(), EXACT.eye(15), EXACT)
    I = ir.to_float(info)
    assert np.abs(ir.to_float(inv - info)).max() <= 1e-30 * np.abs(I).max()
    assert np.abs(ir.to_float(info - info.T)).max() <= 1e-40 * np.abs(I).max()
    assert np.linalg.eigvalsh(I).min() > 0


@pytest.mark.parametrize("name", ["neg_matched_q", "neg_mean_q", "neg_delta_q"])
def test_quaternion_sign_does_not_matter(exact, name):
    """The pose prior and the prior canonicalise the sign of their rotation error; a negated delta_q negates the predicted q_j
    with it, so the IMU rotation residual is unchanged. Same estimate up to the sign of q, same cost and information."""
    a, b = exact[name], exact["nominal"]
    assert a["iterations"] == b["iterations"] and _close(a, b, 1e-14)
    assert abs(a["final_cost"] - b["final_cost"]) <= 1e-14 * b["final_cost"]
    assert np.abs(a["information"] - b["information"]).max() <= 1e-12 * np.abs(b["information"]).max()


@pytest.mark.parametrize("name", ["gf_tilted", "gf_minus_z", "gf_gx_above"])
def test_tangent_basis_does_not_matter(exact, name):
    """Another orthonormal basis of g's tangent plane (Unit3's rotated by 40 deg) gives the same solve."""
    def rotated(g, A):
        b1, b2 = wr._unit3_basis(g, A)
        c, s = A.num(np.cos(0.7)), A.num(np.sin(0.7))
        return tuple(c * x + s * y for x, y in zip(b1, b2)), tuple(c * y - s * x for x, y in zip(b1, b2))
    a, b = wr.solve(wc._with(CASES[name][1], basis=rotated), EXACT), exact[name]
    assert a["iterations"] == b["iterations"] and _close(a, b, 1e-14)
    assert abs(a["final_cost"] - b["final_cost"]) <= 1e-14 * b["final_cost"]
    assert np.abs(a["information"] - b["information"]).max() <= 1e-12 * np.abs(b["information"]).max()


@pytest.mark.parametrize("name", ["gf_g_nonunit", "gf_bref_nonunit", "gf_gx_below"])
def test_direction_lengths_and_the_basis_switch_do_not_matter(exact, name):
    """Only the directions enter the gravity factor, and both sides of |g_x| = 0.9 give the same solve to 1e-11."""
    other = {"gf_g_nonunit": "gf_tilted", "gf_bref_nonunit": "gf_tilted", "gf_gx_below": "gf_gx_above"}[name]
    a, b = exact[name], exact[other]
    assert a["iterations"] == b["iterations"] and _close(a, b, 1e-11)


def test_oracle_refuses_zero_directions(orc):
    p = CASES["gf_tilted"][1]
    for gf in ((5e-2, (0, 0, 0), (0, 0, 1)), (5e-2, (0, 0, 1), (0, 0, 0))):
        with pytest.raises(RuntimeError):
            _oracle(orc, wc._with(p, gravity_factor=gf))
