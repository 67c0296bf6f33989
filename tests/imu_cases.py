"""Edge cases of the IMU row, one generator per edge with the reason it is an edge. Shared by the CPU reference tests and
the device tests. An interval is (dt[n], acc[n,3], gyr[n,3]); a batch is one noise setting plus a list of
(interval, ba, bg), launched together on the device."""
import numpy as np

from imu_reference import KAIST_NOISE

RATE = 200.0
G16 = 16 * 9.80665


def _axis(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v)


def samples(n, seed, omega=(0.02, -0.03, 0.15), force=(0.3, -0.2, 9.8), dt=1.0 / RATE, jitter=0.0, noise=(3.99e-2, 1.56e-2)):
    """n samples of a smooth body-frame rate and specific force plus white noise, so that no entry is an exact zero.
    jitter: relative uniform spread of dt."""
    rng = np.random.RandomState(seed)
    t = np.arange(n) * dt
    dts = np.full(n, dt)
    if jitter:
        dts = dt * (1 + rng.uniform(-jitter, jitter, n))
    w = np.asarray(omega, np.float64)[None, :] * (1 + 0.2 * np.sin(3.0 * t))[:, None]
    f = np.asarray(force, np.float64)[None, :] + 0.5 * np.stack([np.sin(2 * t), np.cos(1.5 * t), np.sin(0.7 * t)], 1)
    gyr = w + rng.normal(0, noise[1], (n, 3))
    acc = f + rng.normal(0, noise[0], (n, 3))
    return dts, acc, gyr


def biases(seed, sa=2e-2, sg=2e-3):
    """Small random accelerometer and gyroscope biases."""
    rng = np.random.RandomState(1000 + seed)
    return rng.normal(0, sa, 3), rng.normal(0, sg, 3)


def _empty():
    return np.zeros(0), np.zeros((0, 3)), np.zeros((0, 3))


def _one(iv, seed, ba=None, bg=None):
    b = biases(seed)
    return (iv, b[0] if ba is None else np.asarray(ba, np.float64), b[1] if bg is None else np.asarray(bg, np.float64))


def _spin(n, rate, axis, seed):
    return samples(n, seed, omega=rate * _axis(axis), force=(0.1, 0.2, 9.8))


def _batch(lengths, seed):
    return [_one(samples(n, seed + k), seed + k) for k, n in enumerate(lengths)]


def _with(iv, k, dt):
    dts, acc, gyr = (a.copy() for a in iv)
    dts[k] = dt
    return dts, acc, gyr


def _saturated(n, seed):
    dts, acc, gyr = samples(n, seed, force=(20.0, -30.0, 9.8))
    acc[::3] = np.sign(acc[::3]) * G16          # readings clipped at the +-16 g full scale
    acc[1::3, 0] = G16
    acc[2::3, 1] = -G16
    return dts, acc, gyr


def batches():
    """name -> (reason, noise4, [(interval, ba, bg), ...])."""
    K = KAIST_NOISE
    b20 = lambda s: _one(samples(20, s), s)
    still = samples(20, 20, noise=(3.99e-2, 0.0))
    return {
        "empty_first": ("an interval with no sample leaves the warp's initial state; first warp of the batch", K,
                        [_one(_empty(), 1), b20(2), b20(3)]),
        "empty_middle": ("an empty interval between two full ones: its neighbours must not see its state", K,
                         [b20(4), _one(_empty(), 5), b20(6)]),
        "empty_last": ("an empty interval as the last of the batch", K, [b20(7), b20(8), _one(_empty(), 9)]),
        "one_sample": ("one sample only latches acc_0 / gyr_0: J = I, P = 0, sum_dt = 0", K, [_one(samples(1, 10), 10)]),
        "two_samples": ("two samples are exactly one mid-point step", K, [_one(samples(2, 11), 11)]),
        "bench_20": ("the bench shape: 20 samples at 200 Hz", K, [b20(12)]),
        "long_2001": ("10 s at 200 Hz: drift of the re-normalisation of delta_q and growth of P", K,
                      [_one(samples(2001, 13), 13)]),
        "jitter30": ("dt with +-30 % jitter", K, [_one(samples(40, 14, jitter=0.3), 14)]),
        "zero_dt": ("a duplicated timestamp: one step with dt = 0", K, [_one(_with(samples(20, 15), 7, dt=0.0), 15)]),
        "tiny_dt": ("dt = 1e-9: F = I to rounding, V ~ 0", K, [_one(_with(samples(20, 16), 9, dt=1e-9), 16)]),
        "gap_half_second": ("a dropped packet: one 0.5 s step", K, [_one(_with(samples(20, 17), 10, dt=0.5), 17)]),
        "spin_12": ("12 rad/s about a tilted axis: large rotation per step", K, [_one(_spin(40, 12.0, (1, 2, 3), 18), 18)]),
        "past_pi": ("the accumulated rotation passes pi: delta_q.w < 0 at the end, no sign canonicalisation", K,
                    [_one(_spin(72, 12.0, (0.3, -0.2, 1.0), 19), 19)]),
        "bg_equals_omega": ("b_g equal to the mean rate: un_gyr ~ 0", K, [_one(still, 20, bg=(0.5 * (still[2][:-1] + still[2][1:])).mean(0))]),
        "ba_half": ("b_a = 0.5 m/s^2 on every axis", K, [_one(samples(20, 21), 21, ba=(0.5, 0.5, 0.5))]),
        "saturated_16g": ("readings clipped at +-16 g", K, [_one(_saturated(20, 22), 22)]),
        "batch_1": ("a batch of one interval", K, _batch([20], 30)),
        "batch_3": ("3 intervals: a partial block of 4 warps", K, _batch([20, 3, 41], 31)),
        "batch_5": ("5 intervals: one full block of 4 warps plus one", K, _batch([7, 20, 1, 0, 33], 32)),
        "batch_37": ("37 intervals of very different lengths: isolation of each warp's shared state", K,
                     _batch([int(n) for n in np.random.RandomState(33).choice([0, 1, 2, 5, 20, 21, 64, 150], 37)], 33)),
        "one_step": ("one 5 ms step: the p rows of V are dt/2 times its v rows, Sigma is singular", K, [_one(samples(2, 39), 39)]),
        "short_5ms": ("5 ms at 1 kHz with a small bias random walk: cond(Sigma) >= 1e10", (KAIST_NOISE[0], KAIST_NOISE[1], 1e-7, 1e-7),
                      [_one(samples(6, 40, dt=1e-3), 40)]),
        "zero_random_walk": ("acc_w = gyr_w = 0: the bias blocks of Sigma are 0, Sigma is not positive definite",
                             (KAIST_NOISE[0], KAIST_NOISE[1], 0.0, 0.0), [_one(samples(20, 41), 41)]),
    }


# ------------------------------------------------------------------ factor cases
def _quat(angle, axis):
    a = _axis(axis)
    return np.concatenate([[np.cos(angle / 2)], np.sin(angle / 2) * a])


SUBMAPS = {
    "identity": ("the submap frame is the local frame", np.array([0, 0, 0, 1.0, 0, 0, 0])),
    "yaw90": ("a 90 deg yaw and a translation", np.concatenate([[4.0, -3.0, 0.5], _quat(np.pi / 2, (0, 0, 1))])),
    "tilt170": ("170 deg about a tilted axis: gravity far from z in the submap frame",
                np.concatenate([[-2.0, 7.0, 1.0], _quat(np.radians(170), (1, -2, 0.5))])),
}


def state_i(seed, ba, bg):
    rng = np.random.RandomState(2000 + seed)
    q = _quat(rng.uniform(-1, 1), rng.normal(size=3))
    return np.concatenate([rng.normal(0, 5, 3), q, rng.normal(0, 2, 3), ba, bg])


def perturbations():
    """name -> (reason, delta15 or 'flip'): where state j sits relative to the prepared start (the prediction)."""
    return {
        "start": ("the prepared start: r ~ 0", np.zeros(15)),
        "moved": ("+-0.3 m, +-0.2 rad, +-0.5 m/s and bias offsets",
                  np.array([0.3, -0.3, 0.2, 0.2, -0.1, 0.15, 0.5, -0.5, 0.3, 0.05, -0.04, 0.03, 5e-3, -4e-3, 3e-3])),
        "flipped": ("q_j negated: e.w < 0, the residual is not sign-canonicalised", "flip"),
    }


MISMATCH = (np.array([0.05, -0.05, 0.05]), np.array([5e-3, -5e-3, 5e-3]))   # state i's biases minus the linearisation biases
WEIGHTS = (0.5, 1.0, 1e3)
