"""Edge cases of the window update (dl_window_optimize_batch), one generator per edge with the reason it is an edge. Shared by
the CPU reference tests and the device tests. A case is a window_reference.problem; intervals are pre-integrated by the fp64
imu_reference (pinned bit for bit to dl_imu_preintegrate), so the device and both references read the same numbers."""
import copy
import ctypes as C

import numpy as np

import imu_cases
import imu_reference as ir
import window_reference as wr

SIGMAS = (0.05, 0.01, 0.5, 1e-2)   # prior sigmas of p, theta, v, biases


def interval(n, seed, **kw):
    """n samples of imu_cases.samples pre-integrated at small random linearisation biases."""
    dts, acc, gyr = imu_cases.samples(n, seed, **kw)
    ba, bg = imu_cases.biases(seed)
    return ir.preintegrate(ir.KAIST_NOISE, ba, bg, dts, acc, gyr)


def prior(seed, sigmas=SIGMAS):
    """Correlated SPD information: diag(1 / sigma^2) plus a random PSD part of 5 % in the scaled entries."""
    s = np.array([sigmas[0]] * 3 + [sigmas[1]] * 3 + [sigmas[2]] * 3 + [sigmas[3]] * 6) if len(sigmas) == 4 else np.asarray(sigmas)
    A = np.random.RandomState(3000 + seed).normal(0, 1, (15, 15))
    d = 1 / s
    return np.diag(d * d) + 0.05 * (A @ A.T) * np.outer(d, d) / 15


def _qmul(a, b):
    return np.array(ir.qmul(tuple(a), tuple(b)))


def _yaw(angle):
    return np.array([np.cos(angle / 2), 0, 0, np.sin(angle / 2)])


def base(seed, n=21, bias_offset=None, matched_offset=(0.01, -0.008, 0.005, 0.004), sigmas=SIGMAS, **kw):
    """A 0.1 s interval (n = 21 samples at 200 Hz), the previous key at the linearisation biases (+ bias_offset), the matched pose
    a little off the IMU prediction. kw: window_reference.problem options."""
    pre = interval(n, seed)
    ba, bg = np.array(pre.ba), np.array(pre.bg)
    if bias_offset is not None:
        ba, bg = ba + bias_offset[0], bg + bias_offset[1]
    mean_i = imu_cases.state_i(seed, ba, bg)
    pred = np.array(ir.predict(mean_i, pre), float)
    z = pred[:7].copy()
    z[:3] += matched_offset[:3]
    z[3:] = _qmul(_yaw(matched_offset[3]), z[3:])
    return wr.problem(mean_i, prior(seed, sigmas), pre, z, **kw)


def _with(p, **kw):
    q = dict(p)
    q.update(kw)
    return q


def _negated_dq(pre):
    pre = copy.copy(pre)
    pre.dq = tuple(-c for c in pre.dq)
    return pre


GF = (5e-2, (0.01, -0.02, 1.0), (0.0, 0.0, 1.0))
SPIN = 12.0 * np.array([0.3, -0.2, 1.0]) / np.linalg.norm([0.3, -0.2, 1.0])   # rad/s


def cases():
    """name -> (reason, problem). Every converged case keeps its step norms half a decade away from the 1e-10 threshold.
    fp64_step_floor marks the cases whose weights are so large (1 / sigma^2 = 1e8, or Sigma^-1 of an ill-conditioned Sigma) that
    an fp64 Gauss-Newton step at the optimum is rounding noise of about 1e-10: there an fp64 solver may take one step more."""
    nominal = base(1)
    far = base(9, matched_offset=(0.3, -0.1, 0.1, np.radians(60)))
    out = {
        "nominal": ("0.1 s KAIST interval, correlated SPD prior", nominal),
        "bias_offset": ("x_i's biases away from the linearisation: the bias correction and its dependence on x_i",
                        base(2, bias_offset=imu_cases.MISMATCH)),
        "short_interval": ("5 samples at 1 kHz: Sigma ill-conditioned (kappa >= 1e10)",
                           _with(base(28), pre=interval(6, 28, dt=1e-3), fp64_step_floor=True)),
        "spin_past_pi": ("1 s at 12 rad/s: delta_q past pi", _with(base(28), pre=interval(201, 28, omega=SPIN))),
        "one_sample": ("one sample: Sigma = 0, not positive definite (termination 2)", _with(base(5), pre=interval(1, 5))),
        "prior_wide": ("prior sigmas from 1e-4 to 1e2", _with(base(6, sigmas=np.logspace(-4, 2, 15)), fp64_step_floor=True)),
        "prior_negated": ("negated prior information: the normal equations are not positive definite (termination 2)",
                          _with(nominal, prior=-nominal["prior"])),
        "neg_matched_q": ("the matched pose's quaternion negated: the pose prior's w < 0 flip",
                          _with(nominal, matched=np.concatenate([nominal["matched"][:3], -nominal["matched"][3:]]))),
        "neg_mean_q": ("the prior mean's quaternion negated: the prior's w < 0 flip",
                       _with(nominal, mean_i=np.concatenate([nominal["mean_i"][:3], -nominal["mean_i"][3:7], nominal["mean_i"][7:]]))),
        "neg_delta_q": ("delta_q negated: the prediction's q_j flips with it, the IMU rotation residual does not",
                        _with(nominal, pre=_negated_dq(nominal["pre"]))),
        "far_iter1": ("matched pose 0.3 m and 60 deg of yaw off, one iteration", _with(far, max_iter=1)),
        "far_iter2": ("the same, two iterations", _with(far, max_iter=2)),
        "far_iter3": ("the same, three iterations", _with(far, max_iter=3)),
        "far_iter0": ("the same, max_num_iterations = 0 (10)", _with(far, max_iter=0)),
        "initial_j": ("initial_j given, off the prediction", _with(nominal, initial_j=_moved(nominal))),
        "neg_initial_j": ("initial_j given with its quaternion negated: the IMU rotation residual starts on the other sheet",
                          _with(nominal, initial_j=_negq(_moved(nominal)))),
        "imu_weight_0.3": ("imu_weight 0.3", base(7, imu_weight=0.3)),
        "imu_weight_3": ("imu_weight 3", base(7, imu_weight=3.0)),
        "gravity_tilted": ("gravity vector tilted off z", base(8, G=(0.3, -0.2, 9.79))),
        "gravity_9.80665": ("standard gravity", base(8, G=(0.0, 0.0, 9.80665))),
        "gf_z": ("gravity factor, g = z", base(28, gravity_factor=(5e-2, (0, 0, 1.0), (0, 0, 1.0)))),
        "gf_minus_z": ("gravity factor, g = -z: R_j b_ref is antiparallel, the residual's Jacobian has rank 0 there",
                       base(28, gravity_factor=(5e-2, (0, 0, -1.0), (0, 0, 1.0)))),
        "gf_tilted": ("gravity factor, tilted g", base(11, gravity_factor=GF)),
        "gf_gx_below": ("|g_x| = 0.9 - 1e-12: the device's basis helper is x", base(28, gravity_factor=_gx(0.9 - 1e-12))),
        "gf_gx_above": ("|g_x| = 0.9 + 1e-12: the device's basis helper is y", base(28, gravity_factor=_gx(0.9 + 1e-12))),
        "gf_g_nonunit": ("g of length 9.8: only its direction counts", base(11, gravity_factor=(GF[0], tuple(9.8 * np.array(GF[1])), GF[2]))),
        "gf_bref_nonunit": ("b_ref of length 2: only its direction counts", base(11, gravity_factor=(GF[0], GF[1], (0.0, 0.0, 2.0)))),
    }
    return out


def _moved(p):
    x = np.array(ir.predict(p["mean_i"], p["pre"]), float)
    x[:3] += [0.02, -0.01, 0.015]
    x[3:7] = _qmul(_yaw(0.02), x[3:7])
    x[7:10] += [0.05, -0.05, 0.02]
    return x


def _negq(x):
    x = x.copy()
    x[3:7] = -x[3:7]
    return x


def _gx(gx):
    """Gravity factor with the unit g = (gx, 0, sqrt(1 - gx^2)): the device picks its tangent basis by |g_x| < 0.9."""
    g = np.array([gx, 0.0, np.sqrt(1 - gx * gx)])
    return (5e-2, tuple(g), (0.0, 0.0, 1.0))


# ------------------------------------------------------------------ device / oracle arguments
def preint_struct(pre, cls):
    """dl_preintegration (dliom.Preintegration or orc.Preintegration) from an fp64 imu_reference.Preintegration."""
    d = lambda v: (C.c_double * len(v))(*[float(x) for x in v])
    return cls(float(pre.sum_dt), d(pre.dp), d(pre.dq), d(pre.dv), d(pre.ba), d(pre.bg), d(np.asarray(pre.J, float).reshape(-1)),
               d(np.asarray(pre.P, float).reshape(-1)))


def options(p):
    """Keyword arguments of Context.window_optimize_batch / window_evaluate and orc.window_optimize (except G / gravity)."""
    return dict(sigma_t=p["sigma_t"], sigma_r=p["sigma_r"], imu_weight=p["imu_weight"], gravity_factor=p["gravity_factor"])


def batch(count, seed):
    """count different problems: 8 intervals of 5 to 40 samples, each member its own previous key, prior and matched pose."""
    pool = [interval(n, seed + k) for k, n in enumerate((5, 11, 21, 40, 17, 8, 33, 26))]
    out = []
    rng = np.random.RandomState(seed)
    for k in range(count):
        pre = pool[k % len(pool)]
        mean_i = imu_cases.state_i(seed * 10000 + k, np.array(pre.ba), np.array(pre.bg))
        z = np.array(ir.predict(mean_i, pre), float)[:7]
        z[:3] += rng.uniform(-0.03, 0.03, 3)
        z[3:] = _qmul(_yaw(rng.uniform(-0.02, 0.02)), z[3:])
        out.append(wr.problem(mean_i, prior(seed * 10000 + k), pre, z))
    return out
