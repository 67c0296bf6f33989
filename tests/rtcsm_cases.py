"""Inputs for the real-time correlative scan matcher, one generator per edge of the device search (dl_rtcsm.cu, its kernels and the
tables of its host part) and of the reference's Match.

Every generator builds a Case and checks, with the numpy reference (rtcsm_reference), that its input sits on the side of the
edge it is named for; the assertion at its end names the edge. Every case but the penalty-underflow ones also checks that no
candidate is exp-ambiguous, so its scores can be demanded bit for bit.

Cases are built on first use (`get(name)`, cached for the session): collecting a test module costs nothing, and a generator
whose self-check fails fails the tests of its own case only. `NAMES` lists every case.
"""
import functools
from dataclasses import dataclass

import numpy as np

import rtcsm_reference as ref

f32 = np.float32
IDENTITY = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
RES = 0.1
POINTS_PER_TILE, LANES, WARPS = 512, 32, 8      # the device's staging tile, strip and CTA shapes


@dataclass
class Case:
    name: str
    grid: ref.SparseGrid
    points: np.ndarray
    pose: np.ndarray
    linear_window: float
    angular_window: float
    w_t: float
    w_r: float
    underflow: bool = False

    @functools.cached_property
    def result(self):
        return ref.match(self.grid, self.points, self.pose, self.linear_window, self.angular_window, self.w_t, self.w_r)

    @property
    def args(self):
        return self.points, self.pose, self.linear_window, self.angular_window, self.w_t, self.w_r


def _case(name, grid, points, pose=IDENTITY, linear=0.15, angular=None, w_t=0.1, w_r=0.1, rotations=1):
    """`angular` None: the window that gives `rotations` (A) at the case's farthest point, exactly A steps."""
    pts = np.asarray(points, f32).reshape(-1, 3)
    if angular is None:
        step = ref.angular_step(grid.resolution, ref.max_scan_range(pts, grid.resolution))
        angular = float(np.float64(step) * rotations)
    c = Case(name, grid, pts, np.asarray(pose, np.float64), linear, angular, w_t, w_r)
    return c


def _checked(c, distinct=True):
    m = c.result
    if not c.underflow:
        assert not m.ambiguous().any(), "exp-ambiguous candidates"
    assert m.best_index >= 0
    if distinct:
        assert len(np.unique(m.scores)) > 1, "every candidate scores the same"
    return c


def _grid(cells, values, resolution=RES):
    return ref.SparseGrid(resolution, np.asarray(cells, np.int64).reshape(-1, 3), np.asarray(values, np.uint16))


def _random_grid(rng, half=(16, 16, 8), density=0.5, resolution=RES):
    b = np.array(half)
    cube = np.stack(np.meshgrid(*[np.arange(-s, s) for s in b], indexing="ij"), -1).reshape(-1, 3)
    cells = cube[rng.random(len(cube)) < density]
    return _grid(cells, rng.integers(1, 32768, len(cells)), resolution)


def _yaw(theta, t=(0.0, 0.0, 0.0)):
    return np.array([*t, np.cos(theta / 2), 0, 0, np.sin(theta / 2)], np.float64)


# ----------------------------------------------------------------------------------------------- cloud sizes
CLOUD_SIZES = (1, 31, 32, 33, 511, 512, 513, 1024, 1025, 2561)


def cloud_size(n):
    """Strip tails (n mod 32), tile tails (n mod 512) and both staging buffers reused twice (2 561 points = 6 tiles)."""
    rng = np.random.default_rng(1000 + n)
    g = _random_grid(rng)
    pts = (rng.uniform(-1, 1, (n, 3)) * [1.4, 1.4, 0.6]).astype(f32)
    c = _checked(_case(f"cloud_{n}", g, pts, _yaw(0.01, (0.013, -0.021, 0.004)), 0.1, rotations=1), distinct=n > 0)
    assert len(c.points) == n and c.result.window.num_rotations == 27
    return c


# ----------------------------------------------------------------------------------------------- candidate shapes
SHAPES = [(0, 0), (0, 1), (1, 0), (1, 1), (2, 1), (3, 1), (1, 2), (2, 2), (3, 2)]   # (L, A)


def shape(L, A):
    """L = 1, 27, 125, 343 translations against R = 1, 27, 125 rotations: L never a multiple of 32, and warps per scan
    R * ceil(L / 32) mostly not a multiple of the CTA's 8; (3, 2) spans 172 CTAs."""
    rng = np.random.default_rng(50 + 7 * L + A)
    g = _random_grid(rng)
    pts = (rng.uniform(-1, 1, (45, 3)) * [1.2, 1.2, 0.5]).astype(f32)
    c = _checked(_case(f"shape_L{L}_A{A}", g, pts, _yaw(-0.02, (0.031, 0.017, -0.012)), L * RES, rotations=A),
                 distinct=L + A > 0)
    w = c.result.window
    assert (w.linear, w.angular) == (L, A)
    return c


# ----------------------------------------------------------------------------------------------- window rounding
def _with_far_point(rng, far, n=40):
    pts = (rng.uniform(-1, 1, (n, 3)) * [1.2, 1.2, 0.5]).astype(f32)
    return np.concatenate([pts, np.asarray(far, f32).reshape(1, 3)])


def linear_half(side):
    """The linear window on a .5 quotient of the float resolution (RoundToInt rounds it away from zero) and one double ulp to
    either side."""
    rng = np.random.default_rng(71)
    g = _random_grid(rng)
    w = 1.5 * float(f32(RES))
    w = {"below": np.nextafter(w, 0.0), "on": w, "above": np.nextafter(w, 1.0)}[side]
    c = _checked(_case(f"linear_half_{side}", g, _with_far_point(rng, [0, 0, 0]), IDENTITY, w, rotations=0))
    q = np.float64(w) / np.float64(f32(RES))
    assert (q < 1.5, q == 1.5, q > 1.5)[["below", "on", "above"].index(side)]
    assert c.result.window.linear == (1 if side == "below" else 2)
    return c


def floor(side):
    """The farthest point one float ulp inside / beyond the 3 * resolution floor of max_scan_range, the angular window between
    the two steps' multiples so that A differs."""
    r3 = f32(3.0) * f32(RES)
    far = {"inside": np.nextafter(r3, f32(0)), "beyond": np.nextafter(r3, f32(1))}[side]
    pts = np.array([[0.05, 0.02, 0.0], [-0.1, 0.05, 0.03], [far, 0, 0], [0.0, -0.12, 0.1]], f32)
    g = _random_grid(np.random.default_rng(72), (6, 6, 6), 0.8)
    s_in, s_out = ref.angular_step(RES, r3), ref.angular_step(RES, np.nextafter(r3, f32(1)))
    assert s_out < s_in
    ang = float(np.float64(s_in) * 1.5 + (np.float64(s_out) - np.float64(s_in)) * 0.75)    # near 1.5 steps, between the two
    c = _checked(_case(f"floor_{side}", g, pts, IDENTITY, 0.1, ang))
    w = c.result.window
    assert w.max_scan_range == (r3 if side == "inside" else far)
    return c


CLIFF = f32(4096.0) * f32(RES)


def far_point(where):
    """A farthest point between 200 m and the acosf cliff (the angular window is wider there than at 200 m), and one beyond
    the cliff (step 0, RoundToInt(+inf) = 0: one rotation)."""
    rng = np.random.default_rng(73)
    g = _random_grid(rng)
    d = {"250m": 250.0, "beyond_cliff": 500.0}[where]
    far = np.array([d * 0.6, -d * 0.8, 0.0], f32)
    c = _checked(_case(f"far_{where}", g, _with_far_point(rng, far), _yaw(0.005), 0.1, np.deg2rad(0.1)))
    w = c.result.window
    if where == "250m":
        at200 = ref.window(np.array([[200, 0, 0]], f32), RES, 0.0, np.deg2rad(0.1))
        assert w.angular == 5 and at200.angular == 4 and w.max_scan_range < CLIFF
    else:
        assert w.step == 0 and w.angular == 0 and w.max_scan_range > CLIFF
    return c


# ----------------------------------------------------------------------------------------------- cell boundaries
def _boundary_points(transform_x, centre_shift, targets, resolution=RES, spread=256):
    """x coordinates whose centre-candidate transform (`transform_x`, float), divided by the float resolution, lies within 4 ulp
    of k + 1/2 (on it where representable) for every k in `targets`; also how many of them a reciprocal multiply rounds to the
    other integer."""
    r = f32(resolution)
    out, flips = [], 0
    for k in targets:
        half = f32(abs(k) + 0.5) * f32(1 if k >= 0 else -1)
        lo = hi = f32(np.float64(half) * np.float64(r) - centre_shift)
        cand = [lo]
        for _ in range(spread):
            lo, hi = np.nextafter(lo, f32(-np.inf)), np.nextafter(hi, f32(np.inf))
            cand += [lo, hi]
        cand = np.array(cand, f32)
        wx = transform_x(cand)
        q = wx / r
        near = np.abs(q.astype(np.float64) - np.float64(half)) <= 4 * np.float64(np.spacing(np.abs(half)))
        assert near.any(), k
        flips += int((ref.round_to_int(wx[near] * (f32(1) / r)) != ref.round_to_int(q[near])).sum())
        out.append(cand[near])
    return np.concatenate(out), flips


BOUNDARY_TARGETS = (0, 3, -4, 6, -8, 10, 15, -19, 23)


def boundary(kind):
    """Centre-candidate x coordinates within 4 ulp of k + 1/2, positive and negative, y = z = 0; `identity` with the identity
    initial pose, `posed` with a translated one. Some of them round to the other integer through the reciprocal multiply,
    which the device must not take there."""
    rng = np.random.default_rng(80)
    g = _random_grid(rng, (26, 4, 4), 0.9)
    pose = IDENTITY if kind == "identity" else np.array([0.0123, 0.0, 0.0, 1, 0, 0, 0])
    t, q = ref.float_pose(pose)
    cq = ref.normalized(ref.qmul(q, np.array([1, 0, 0, 0], f32)))
    ct = ref.rotate(q, np.zeros((1, 3), f32))[0] + t

    def tx(x):
        return (ref.rotate(cq, np.column_stack([x, np.zeros_like(x), np.zeros_like(x)]).astype(f32)) + ct)[:, 0]

    xs, flips = _boundary_points(tx, float(t[0]), BOUNDARY_TARGETS)
    pts = np.column_stack([xs, np.zeros((len(xs), 2))]).astype(f32)
    c = _checked(_case(f"boundary_{kind}", g, pts, pose, 0.1, 0.0))
    assert flips > 0, "no point where the reciprocal rounds differently"
    return c


def boundary_large():
    """Coordinates near |x / resolution| = 2^22 cells, where the device's rounding switches from the reciprocal to the
    division, on .5 boundaries (exact there: the float spacing is 0.5 or 0.25), positive and negative. Those cells are far
    outside any grid and read 0.1; the other points see the grid."""
    rng = np.random.default_rng(81)
    g = _random_grid(rng, (12, 12, 6), 0.9)
    r = f32(RES)
    big = []
    for q in (4194303.5, 4194304.5, 4194302.5, 4194305.0):
        for s in (1, -1):
            x = f32(q * s) * r
            big.append([x, 0.0, 0.0])
    near = (rng.uniform(-1, 1, (30, 3)) * [1.0, 1.0, 0.4]).astype(f32)
    c = _checked(_case("boundary_2^22", g, np.concatenate([near, np.array(big, f32)]), IDENTITY, 0.1, rotations=0))
    assert c.result.window.max_scan_range > f32(400000)
    return c


def outside_grid():
    """Negative coordinates and points outside the grid's cells, where absent cells read 0.1."""
    rng = np.random.default_rng(82)
    g = _random_grid(rng, (8, 8, 4), 0.7)
    pts = np.concatenate([(rng.uniform(-1, 0, (20, 3)) * [0.8, 0.8, 0.4]).astype(f32),
                          (rng.uniform(-1, 1, (20, 3)) * [30, 30, 5]).astype(f32)])
    c = _checked(_case("outside_grid", g, pts, _yaw(0.03, (-0.2, 0.1, 0.0)), 0.2, rotations=1))
    return c


# ----------------------------------------------------------------------------------------------- cell values
def all_values():
    """Values 1..32 767 in a 32^3 cube; one point at the origin, zero weights: the 35 937 translations read every value."""
    cube = np.stack(np.meshgrid(*[np.arange(-16, 16)] * 3, indexing="ij"), -1).reshape(-1, 3)[1:]
    g = _grid(cube, np.arange(1, 32768))
    c = _checked(_case("all_values", g, np.zeros((1, 3), f32), IDENTITY, 1.6, 0.0, 0.0, 0.0))
    m = c.result
    assert m.window.linear == 16
    ax = np.arange(-16, 17)
    zyx = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    seen = g.lookup(zyx[:, ::-1])
    assert set(seen.tolist()) == set(range(32768))
    assert np.array_equal(m.scores, ref.PROBABILITY[seen])
    return c


# ----------------------------------------------------------------------------------------------- ties
def empty_grid():
    """No cell at all and zero weights: every one of 343 * 27 candidates (38 CTAs) reads 0.1 at every point, so all scores
    are equal and index 0 must win."""
    rng = np.random.default_rng(90)
    pts = (rng.uniform(-1, 1, (70, 3)) * [2, 2, 1]).astype(f32)
    c = _checked(_case("tie_empty_grid", _grid(np.zeros((0, 3)), []), pts, _yaw(0.1, (1, 2, 0.5)), 0.3, w_t=0.0, w_r=0.0,
                       rotations=1), distinct=False)
    m = c.result
    assert len(np.unique(m.scores)) == 1 and m.best_index == 0 and m.num_candidates == 343 * 27
    return c


def _where(index, R, L):
    """(CTA, warp task) of candidate index l * R + r for one scan."""
    l, r = divmod(index, R)
    chunks = (L + LANES - 1) // LANES
    task = r * chunks + l // LANES
    return task // WARPS, task


def symmetric(relation):
    """A grid symmetric under one mirror and a cloud on the mirror plane: mirrored translations tie exactly with non-zero
    weights, and the lower index must win. The mirror and the peak are chosen so that the two tied candidates run in the same
    warp, in two warps of one CTA, or in two CTAs."""
    L = 5
    n = 2 * L + 1
    rng = np.random.default_rng(91)
    for axis in (0, 1, 2):
        for d in range(1, L + 1):
            for u in range(-L, L + 1):
                peak = np.zeros(3, np.int64)
                peak[axis] = d
                peak[(axis + 1) % 3] = u
                mirror = peak.copy()
                mirror[axis] = -d
                idx = [((p[2] + L) * n + (p[1] + L)) * n + (p[0] + L) for p in (peak, mirror)]
                (c0, t0), (c1, t1) = (_where(i, 1, n ** 3) for i in idx)
                ok = {"warp": t0 == t1, "cta": t0 != t1 and c0 == c1, "ctas": c0 != c1}[relation]
                if ok:
                    break
            else:
                continue
            break
        else:
            continue
        break
    else:
        raise AssertionError(relation)
    # cells symmetric under the mirror: random low values, the peak pair high
    cube = np.stack(np.meshgrid(*[np.arange(-L - 1, L + 2)] * 3, indexing="ij"), -1).reshape(-1, 3)
    vals = rng.integers(1, 8000, len(cube))
    key = {tuple(c): v for c, v in zip(cube, vals)}
    for c in cube:
        m = c.copy()
        m[axis] = -m[axis]
        key[tuple(c)] = key[tuple(m)] = min(key[tuple(c)], key[tuple(m)])
    key[tuple(peak)] = key[tuple(mirror)] = 30000
    cells = np.array(list(key.keys()))
    g = _grid(cells, list(key.values()))
    c = _checked(_case(f"tie_{relation}", g, np.zeros((1, 3), f32), IDENTITY, L * RES, 0.0, 0.1, 0.1))
    m = c.result
    assert sorted(m.tied().tolist()) == sorted(idx) and m.best_index == min(idx)
    return c


def mirrored_cloud():
    """The ±x-symmetric grid with a cloud in the x = 0 plane and rotations: the best score is tied, the lowest index wins."""
    rng = np.random.default_rng(92)
    cube = np.stack(np.meshgrid(np.arange(-8, 9), np.arange(-8, 8), np.arange(-4, 4), indexing="ij"), -1).reshape(-1, 3)
    key = {}
    for c in cube:
        a = (abs(int(c[0])), int(c[1]), int(c[2]))
        key.setdefault(a, int(rng.integers(1, 32768)))
    g = _grid(cube, [key[(abs(int(c[0])), int(c[1]), int(c[2]))] for c in cube])
    pts = np.column_stack([np.zeros(30), rng.uniform(-0.6, 0.6, 30), rng.uniform(-0.3, 0.3, 30)]).astype(f32)
    c = _checked(_case("tie_mirrored_cloud", g, pts, IDENTITY, 0.2, 0.0, 0.1, 0.1))
    assert len(c.result.tied()) >= 2
    return c


# ----------------------------------------------------------------------------------------------- penalty underflow
def underflow():
    """Weights so large that exp(-(a * a)) takes most scores into float denormals and many to 0: the denormals must survive
    (the build keeps them: -ftz=false), the zeros never win. The reference would CHECK-fail only if every score were 0."""
    rng = np.random.default_rng(95)
    g = _random_grid(rng)
    pts = (rng.uniform(-1, 1, (60, 3)) * [1.2, 1.2, 0.5]).astype(f32)
    c = _case("penalty_underflow", g, pts, _yaw(0.01), 0.2, w_t=29.0, w_r=1.0, rotations=1)
    c.underflow = True
    _checked(c)
    s = c.result.scores
    tiny = np.finfo(f32).tiny
    assert ((s > 0) & (s < tiny)).sum() > 20 and (s == 0).sum() > 20 and (s >= tiny).sum() > 0
    return c


# ----------------------------------------------------------------------------------------------- initial pose
def large_translation():
    """A non-trivial initial pose far from the origin (700 m, cells near 7 000): the float cast of `initial` decides the
    candidates' translations."""
    rng = np.random.default_rng(97)
    pose = np.array([700.123456789, -650.987654321, 30.5, 0, 0, 0, 0])
    q = np.array([0.9, 0.1, -0.2, 0.3])
    pose[3:] = q / np.linalg.norm(q)
    pts = (rng.uniform(-1, 1, (200, 3)) * [3, 3, 1]).astype(f32)
    t, qf = ref.float_pose(pose)
    world = ref.rotate(qf, pts) + t
    cells = np.unique(ref.round_to_int(world / f32(RES)), axis=0)
    box = np.concatenate([cells + o for o in np.stack(np.meshgrid(*[np.arange(-2, 3)] * 3, indexing="ij"), -1).reshape(-1, 3)])
    box = np.unique(box, axis=0)
    g = _grid(box, rng.integers(1, 32768, len(box)))
    c = _checked(_case("initial_far", g, pts, pose, 0.2, rotations=1))
    assert np.float64(f32(pose[0])) != pose[0]
    return c


# ----------------------------------------------------------------------------------------------- scenes
def scene(beams, k=0):
    """An adaptive-filtered cloud of a synthetic drive (helpers.workload) on its high-resolution submap, the stock windows."""
    import orc
    from helpers import workload
    w = workload(beams=beams) if beams == 16 else workload(beams=64, num_map_scans=6, num_scans=3)
    g = ref.SparseGrid.from_export(w["hi"].resolution, w["hi"].export())
    ing = orc.ingest_scan(w["opts"], w["scans"][k], w["origin"], w["prev"][k], w["cur"][k])
    keep, _ = orc.adaptive_voxel_filter(ing["returns_tracking"], 2.0, 150, 15.0)
    c = _checked(_case(f"scene{beams}_{k}", g, ing["returns_tracking"][keep], w["cur"][k], 0.15, np.deg2rad(1.0), 0.1, 0.1))
    assert c.result.window.linear == 1 and c.result.window.angular >= 2
    return c


def _registry():
    r = {}
    for n in CLOUD_SIZES:
        r[f"cloud_{n}"] = functools.partial(cloud_size, n)
    for L, A in SHAPES:
        r[f"shape_L{L}_A{A}"] = functools.partial(shape, L, A)
    for side in ("below", "on", "above"):
        r[f"linear_half_{side}"] = functools.partial(linear_half, side)
    for side in ("inside", "beyond"):
        r[f"floor_{side}"] = functools.partial(floor, side)
    for where in ("250m", "beyond_cliff"):
        r[f"far_{where}"] = functools.partial(far_point, where)
    for kind in ("identity", "posed"):
        r[f"boundary_{kind}"] = functools.partial(boundary, kind)
    r["boundary_2^22"], r["outside_grid"], r["all_values"] = boundary_large, outside_grid, all_values
    r["tie_empty_grid"], r["tie_mirrored_cloud"] = empty_grid, mirrored_cloud
    for rel in ("warp", "cta", "ctas"):
        r[f"tie_{rel}"] = functools.partial(symmetric, rel)
    r["penalty_underflow"], r["initial_far"] = underflow, large_translation
    r["scene16_0"] = functools.partial(scene, 16, 0)
    r["scene64_0"] = functools.partial(scene, 64, 0)
    return r


REGISTRY = _registry()
NAMES = list(REGISTRY)
BOUNDARY = ["boundary_identity", "boundary_posed", "boundary_2^22"]


@functools.lru_cache(maxsize=None)
def get(name):
    c = REGISTRY[name]()
    assert c.name == name
    return c
