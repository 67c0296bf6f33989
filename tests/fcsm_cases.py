"""Inputs for the loop-closure coarse matcher, one generator per edge of the device search (dl_fcsm.cu) and of the
reference's MatchWith3DofInitial.

Every generator builds a Case and checks, with the numpy reference (fcsm_reference), that its input sits on the side of the
edge it is named for; the assertion at its end names the edge. `path` is the device search the case must take: "pruned"
(the search index of the high-resolution grid exists and the window has at most 60 000 blocks of 8^3 leaves) or
"exhaustive".

Cases are built on first use (`get(name)`, cached for the session): collecting a test module costs nothing, and a generator
whose self-check fails fails the tests of its own case only. `NAMES` lists every case; `NOT_SMALL` those too large for the
literal branch and bound, `NOT_IN_ORACLE` those the reference itself cannot run.
"""
import functools
from dataclasses import dataclass

import numpy as np

import fcsm_reference as ref
import range_data_inserter_reference as rdi

f32 = np.float32
IDENTITY = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
MAX_BLOCKS = 60000
MAX_INDEX_BYTES = 3 << 30


@dataclass
class Case:
    name: str
    hi: ref.SparseGrid
    lo: ref.SparseGrid
    hi_points: np.ndarray
    lo_points: np.ndarray
    pose: np.ndarray
    min_score: float
    xy_window: float
    z_window: float
    min_low: float
    path: str = "pruned"

    def run(self, all_ties=True):
        return ref.match_3dof(self.hi, self.lo, self.hi_points, self.lo_points, self.pose, self.min_score, self.xy_window,
                              self.z_window, self.min_low, all_ties=all_ties)

    @property
    def small(self):
        """Small enough for the literal branch and bound and the oracle's."""
        wxy, wz = ref.window(self.xy_window, self.z_window, self.hi.resolution)
        return (2 * wxy + 1) ** 2 * (2 * wz + 1) <= 40000 and len(self.hi_points) <= 64 and len(self.hi.cells) <= 40000


def index_bytes(grid):
    """Size of the device's search index of `grid` (bounding box of its bricks, one brick of margin below); 0 when empty."""
    if len(grid.cells) == 0:
        return 0
    b = (grid.cells + rdi.LIMIT) >> 3
    dim = (b.max(axis=0) - b.min(axis=0) + 1) * 8 + 8
    return int(np.prod(dim))


def num_blocks(wxy, wz):
    bxy = (2 * wxy + 1 + 7) // 8
    return bxy * bxy * ((2 * wz + 1 + 7) // 8)


def expected_path(hi, xy_window, z_window):
    wxy, wz = ref.window(xy_window, z_window, hi.resolution)
    ok = 0 < index_bytes(hi) <= MAX_INDEX_BYTES and num_blocks(wxy, wz) <= MAX_BLOCKS
    return "pruned" if ok else "exhaustive"


def _case(name, hi, lo, hi_points, lo_points, pose, min_score, xy_window, z_window, min_low):
    c = Case(name, hi, lo, np.asarray(hi_points, f32).reshape(-1, 3), np.asarray(lo_points, f32).reshape(-1, 3),
             np.asarray(pose, np.float64), min_score, xy_window, z_window, min_low)
    c.path = expected_path(hi, xy_window, z_window)
    return c


def _grid(resolution, cells, values):
    return ref.SparseGrid(resolution, np.asarray(cells, np.int64).reshape(-1, 3), np.asarray(values, np.uint16))


def _yaw(theta, t=(0.0, 0.0, 0.0)):
    return np.array([*t, np.cos(theta / 2), 0, 0, np.sin(theta / 2)], np.float64)


def _scatter(seed, n_hi=64, n_lo=64, box=(20, 20, 6), density=0.25):
    """A random high-resolution grid (0.1 m) of every kind of value, a random low-resolution grid (0.3 m) and clouds inside."""
    rng = np.random.default_rng(seed)
    b = np.array(box)
    grid = np.stack(np.meshgrid(*[np.arange(-s, s) for s in b], indexing="ij"), -1).reshape(-1, 3)
    cells = grid[rng.random(len(grid)) < density]
    hi = _grid(0.1, cells, rng.integers(1, 32768, len(cells)))
    lgrid = np.stack(np.meshgrid(*[np.arange(-(s // 3) - 2, s // 3 + 2) for s in b], indexing="ij"), -1).reshape(-1, 3)
    lcells = lgrid[rng.random(len(lgrid)) < 0.6]
    lo = _grid(0.3, lcells, rng.integers(1, 32768, len(lcells)))
    hp = (rng.uniform(-1, 1, (n_hi, 3)) * b * 0.1 * 0.8).astype(f32)
    lp = (rng.uniform(-1, 1, (n_lo, 3)) * b * 0.1 * 0.8).astype(f32)
    return hi, lo, hp, lp


def _exact_gate(c):
    """Sets min_low to the answer's own low-resolution score (the gate's >= edge); returns the case."""
    m = c.run(all_ties=False)
    assert m.found
    c.min_low = float(m.low_resolution_score)
    m2 = c.run(all_ties=False)
    assert m2.found and m2.offset == m.offset and np.float64(m2.low_resolution_score) == c.min_low   # passes at equality
    return c


# ----------------------------------------------------------------------------------------------- cloud sizes
CLOUD_SIZES = [(n, 64) for n in (1, 3, 4, 5, 1023, 1024, 1025, 2049)] + [(64, n) for n in (1, 1024, 1025, 3000)]


def cloud_size(n_hi, n_lo):
    """n_hi across the 4 point groups and the 1 024-point tiles, n_lo across the gate's tiles; the gate sits at its edge."""
    hi, lo, hp, lp = _scatter(100 + n_hi + 7 * n_lo, n_hi, n_lo)
    c = _exact_gate(_case(f"cloud_hi{n_hi}_lo{n_lo}", hi, lo, hp, lp, _yaw(0.1, (0.05, -0.03, 0.02)), 0.1, 0.8, 0.4, 0.0))
    assert len(c.hi_points) == n_hi and len(c.lo_points) == n_lo
    return c


# ----------------------------------------------------------------------------------------------- brick rows
def _brick_x(x):
    return (x + rdi.LIMIT) >> 3


def brick_rows(phase):
    """Occupied and absent bricks alternate along x; every point's runs of 8 leaves start at `phase` inside a brick row, so
    the run's first row (p0) is absent while the second (p1) is present, and the reverse."""
    rng = np.random.default_rng(200 + phase)
    wxy, wz = 12, 2
    xs = np.arange(-48, 48)
    xs = xs[_brick_x(xs) % 2 == 0]
    grid = np.stack(np.meshgrid(xs, np.arange(-4, 4), np.arange(-3, 3), indexing="ij"), -1).reshape(-1, 3)
    hi = _grid(0.1, grid, rng.integers(1, 32768, len(grid)))
    cx = np.array([-24, -8, 8]) + (wxy + phase) % 8
    hp = np.stack([cx, [1, -2, 0], [0, 1, -1]], 1).astype(f32) * f32(0.1)
    lo = _grid(0.5, np.zeros((1, 3)), [20000])
    c = _case(f"brick_rows_phase{phase}", hi, lo, hp, hp, IDENTITY, 0.1, wxy * 0.1, wz * 0.1, 0.0)
    cells = ref.discretize(hp, IDENTITY, hi.resolution)
    assert ((cells[:, 0] - wxy) & 7 == phase).all()
    occupied = set(_brick_x(xs).tolist())
    runs = [(int(x + o - phase), int(x + o - phase + 8)) for x in cells[:, 0] for o in range(-wxy, wxy + 1, 8)]
    kinds = {(_brick_x(a) in occupied, _brick_x(b) in occupied) for a, b in runs}
    assert (False, True) in kinds and (True, False) in kinds          # p0 absent / p1 present, and the reverse
    return c


# ----------------------------------------------------------------------------------------------- grid edges and the index
def grid_edge_small():
    """A grid at bits 1 (cells in [-64, 64)) with data in its corners; the windows reach past its edges."""
    rng = np.random.default_rng(300)
    corner = np.stack(np.meshgrid(np.arange(58, 64), np.arange(58, 64), np.arange(-64, -59), indexing="ij"), -1).reshape(-1, 3)
    cells = np.concatenate([corner, -corner - 1])
    hi = _grid(0.1, cells, rng.integers(1, 32768, len(cells)))
    hp = np.array([[6.1, 6.0, -6.2], [-6.2, -6.1, 6.1], [6.2, 5.9, -6.1]], f32)
    lo = _grid(0.5, np.zeros((1, 3)), [20000])
    c = _case("grid_edge_bits1", hi, lo, hp, hp, IDENTITY, 0.1, 1.0, 0.6, 0.0)
    assert rdi.bits_for(cells) == 1
    pc = ref.discretize(hp, IDENTITY, hi.resolution)
    assert (pc.max(axis=0) + 10 > 63).any() and (pc.min(axis=0) - 10 < -64).any()
    return c


def grid_edge_large():
    """A grid grown to bits 8 by cells at -8 192 and 8 191; the window reaches past both ends."""
    rng = np.random.default_rng(301)
    xs = np.concatenate([np.arange(-8192, -8180), np.arange(8180, 8192)])
    cells = np.stack(np.meshgrid(xs, np.arange(-3, 3), np.arange(-2, 2), indexing="ij"), -1).reshape(-1, 3)
    hi = _grid(0.1, cells, rng.integers(1, 32768, len(cells)))
    hp = np.array([[-819.0, 0.1, 0.0], [818.9, -0.1, 0.1]], f32)
    lo = _grid(0.5, np.zeros((1, 3)), [20000])
    c = _case("grid_edge_bits8", hi, lo, hp, hp, IDENTITY, 0.1, 1.2, 0.3, 0.0)
    assert rdi.bits_for(cells) == 8 and cells.min() == -8192 and cells.max() == 8191
    pc = ref.discretize(hp, IDENTITY, hi.resolution)
    assert pc[:, 0].min() - 12 < -8192 and pc[:, 0].max() + 12 > 8191 and c.path == "pruned"
    return c


def axis_8000():
    """Data along x at +-8 000 cells: an index of about 16 000 x 24 x 24 bytes, large but built."""
    rng = np.random.default_rng(302)
    xs = np.concatenate([np.arange(-8004, -7996), np.arange(7996, 8004)])
    cells = np.stack(np.meshgrid(xs, np.arange(-4, 4), np.arange(-2, 2), indexing="ij"), -1).reshape(-1, 3)
    hi = _grid(0.1, cells, rng.integers(1, 32768, len(cells)))
    hp = np.array([[800.0, 0.0, 0.0], [799.7, 0.2, 0.1], [-799.9, 0.1, 0.0]], f32)
    lo = _grid(0.5, np.zeros((1, 3)), [20000])
    c = _case("axis_8000", hi, lo, hp, hp, IDENTITY, 0.1, 0.8, 0.3, 0.0)
    assert 64 << 20 > index_bytes(hi) > 4 << 20 and c.path == "pruned"
    return c


def far_corners():
    """Data at two far corners: the index would exceed 3 GiB, the search stays exhaustive."""
    rng = np.random.default_rng(303)
    block = np.stack(np.meshgrid(*[np.arange(0, 4)] * 3, indexing="ij"), -1).reshape(-1, 3)
    cells = np.concatenate([block - 8000, block + 7996])
    hi = _grid(0.1, cells, rng.integers(1, 32768, len(cells)))
    hp = np.array([[-799.9, -799.8, -799.9], [799.8, 799.8, 799.9]], f32)
    lo = _grid(0.5, np.zeros((1, 3)), [20000])
    c = _case("far_corners", hi, lo, hp, hp, IDENTITY, 0.1, 0.6, 0.6, 0.0)
    assert index_bytes(hi) > MAX_INDEX_BYTES and c.path == "exhaustive"
    return c


def margin_brick():
    """The best leaf puts the only point on a cell at a brick start; its block's first offset puts the point 4 cells below
    that brick, inside the index's margin brick. A weaker cell elsewhere makes another block's bound non-zero."""
    hi = _grid(0.1, [[0, 0, 0], [16, 0, 0]], [32767, 9000])
    hp = np.zeros((1, 3), f32)
    lo = _grid(0.5, np.zeros((1, 3)), [20000])
    c = _case("margin_brick", hi, lo, hp, hp, IDENTITY, 0.05, 2.0, 0.3, 0.0)
    m = c.run()
    wxy, wz = m.wxy, m.wz
    assert m.offset == (0, 0, 0) and ((hi.cells[0] + rdi.LIMIT) % 8 == 0).all()            # a brick start
    first = -wxy + 8 * ((0 + wxy) // 8)
    assert 1 <= 0 - first <= 7 and ref.LUT[9000] > 0                                        # 1..7 cells below it
    return c


# ----------------------------------------------------------------------------------------------- windows
# half-widths 0, and 8k - 1, 8k, 8k + 1 (sides 2w + 1 on both sides of a multiple of 8 and on it plus one)
WINDOWS = [(0.0, 0.0, (0, 0)), (0.04, 0.3, (0, 3)), (0.5, 0.049, (5, 0)), (0.7, 0.3, (7, 3)), (0.8, 0.4, (8, 4)), (0.9, 0.5, (9, 5)),
           (1.5, 0.7, (15, 7)), (1.6, 0.8, (16, 8)), (1.7, 0.9, (17, 9))]


def window_case(xy, z, want):
    hi, lo, hp, lp = _scatter(400, 32, 32)
    c = _case(f"window_{want[0]}_{want[1]}", hi, lo, hp, lp, _yaw(-0.05, (0.02, 0.01, -0.03)), 0.1, xy, z, 0.0)
    assert ref.window(xy, z, hi.resolution) == want
    return c


def block_limit(wxy):
    """wxy 399 / wz 20: exactly 60 000 blocks (pruned); wxy 400: 61 206 blocks (exhaustive). 26 M leaves either way."""
    rng = np.random.default_rng(500 + wxy)
    cells = rng.integers(-400, 400, (200, 3)) * [1, 1, 0] + rng.integers(-20, 20, (200, 1)) * [0, 0, 1]
    hi = _grid(0.1, cells, rng.integers(1, 32768, len(cells)))
    hp = (rng.uniform(-1, 1, (6, 3)) * [2.0, 2.0, 0.5]).astype(f32)
    lo = _grid(0.5, np.zeros((1, 3)), [20000])
    r = float(f32(0.1))
    c = _case(f"block_limit_{wxy}", hi, lo, hp, hp, IDENTITY, 0.2, wxy * r, 20 * r, 0.0)
    assert ref.window(c.xy_window, c.z_window, 0.1) == (wxy, 20)
    assert num_blocks(wxy, 20) == {399: 60000, 400: 61206}[wxy]
    assert c.path == ("pruned" if wxy == 399 else "exhaustive")
    return c


WINDOW_TIES = [(res, k, side) for res in (0.05, 0.1, 0.15) for k in (4, 7) for side in ("tie", "below", "above")]


def window_tie(res, k, side):
    """A window whose window / float(resolution) is exactly k + 0.5 (rounds away from zero), or one double below or above."""
    hi, lo, hp, lp = _scatter(600, 16, 16)
    r = float(f32(res))
    h = _grid(res, hi.cells, hi.values)
    tie = (k + 0.5) * r
    for step in range(-4, 5):
        cand = tie
        for _ in range(abs(step)):
            cand = np.nextafter(cand, np.inf if step > 0 else -np.inf)
        if cand / r == k + 0.5:
            tie = float(cand)
            break
    assert tie / r == k + 0.5
    xy = tie
    if side == "below":
        while xy / r >= k + 0.5:
            xy = float(np.nextafter(xy, -np.inf))
    if side == "above":
        while xy / r <= k + 0.5:
            xy = float(np.nextafter(xy, np.inf))
    c = _case(f"window_tie_{res}_{k}_{side}", h, lo, hp, lp, IDENTITY, 0.1, xy, 2.5 * r, 0.0)
    assert ref.window(xy, 2.5 * r, res)[0] == (k if side == "below" else k + 1)
    return c


# ----------------------------------------------------------------------------------------------- ties
def all_leaves_equal():
    """No point reaches a cell: every leaf scores 0.1; min_score 0.05 keeps them all; the lowest index wins."""
    hi = _grid(0.1, [[200, 200, 50]], [32767])
    hp = np.array([[0.0, 0.0, 0.0], [0.3, -0.2, 0.1]], f32)
    lo = _grid(0.5, np.zeros((1, 3)), [20000])
    c = _case("all_leaves_0.1", hi, lo, hp, hp, IDENTITY, 0.05, 0.8, 0.3, 0.0)
    m = c.run()
    assert (m.scores == f32(0.1)).all() and m.offset == (-m.wxy, -m.wxy, -m.wz)
    return c


def symmetric_ties():
    """One point, four equal cells around it: four best leaves; the one of lowest (z, y, x) index wins."""
    hi = _grid(0.1, [[3, 0, 0], [-3, 0, 0], [0, 3, 0], [0, -3, 0]], [32767] * 4)
    hp = np.zeros((1, 3), f32)
    lo = _grid(0.5, np.zeros((1, 3)), [20000])
    c = _case("symmetric_ties", hi, lo, hp, hp, IDENTITY, 0.1, 0.6, 0.2, 0.0)
    m = c.run()
    assert len(m.tied) == 4 and m.offset == (0, -3, 0)
    return c


def tie_gate():
    """Two best leaves; the one of lower index fails the gate, the other passes."""
    hi = _grid(0.1, [[-4, 0, 0], [4, 0, 0]], [32767] * 2)
    hp = np.zeros((1, 3), f32)
    lo = _grid(0.5, [[1, 0, 0]], [32767])
    c = _case("tie_gate", hi, lo, hp, hp, IDENTITY, 0.1, 0.6, 0.2, 0.5)
    m = c.run()
    assert m.offset == (4, 0, 0) and [m.offset_of(i) for i in m.rejected] == [(-4, 0, 0)]
    return c


@functools.lru_cache(maxsize=None)
def at_min_score():
    """min_score equal to the best leaf's score: strictly above it is required, nothing is found; one float below, the best
    leaf is."""
    hi, lo, hp, lp = _scatter(700, 24, 24)
    c = _case("at_min_score", hi, lo, hp, lp, IDENTITY, 0.0, 0.6, 0.3, 0.0)
    best = c.run(all_ties=False)
    c.min_score = float(best.score)
    below = _case("below_min_score", hi, lo, hp, lp, IDENTITY, float(np.nextafter(best.score, f32(0))), 0.6, 0.3, 0.0)
    assert not c.run().found and below.run().offset == best.offset
    return [c, below]


@functools.lru_cache(maxsize=None)
def at_min_low():
    """min_low_resolution_score equal to the answer's low-resolution score (>=); a hair above it, the answer moves."""
    hi, lo, hp, lp = _scatter(701, 24, 40)
    c = _exact_gate(_case("at_min_low", hi, lo, hp, lp, _yaw(0.2), 0.1, 0.6, 0.3, 0.0))
    above = _case("above_min_low", hi, lo, hp, lp, _yaw(0.2), 0.1, 0.6, 0.3, float(np.nextafter(c.min_low, 1.0)))
    assert above.run().offset != c.run().offset
    return [c, above]


def _block_bounds(c, m):
    """Bound of every 8^3 block: sum over points of the largest 8-bit value the point meets inside the block (brute force)."""
    cells = ref.discretize(c.hi_points, c.pose, c.hi.resolution)
    per = [ref.window_sums(c.hi, cell[None], m.wxy, m.wz) for cell in cells]
    side, depth = 2 * m.wxy + 1, 2 * m.wz + 1
    bxy, bz = (side + 7) // 8, (depth + 7) // 8
    out = np.zeros((bz, bxy, bxy), np.int64)
    for p in per:
        for z in range(bz):
            for y in range(bxy):
                for x in range(bxy):
                    out[z, y, x] += p[8 * z:8 * z + 8, 8 * y:8 * y + 8, 8 * x:8 * x + 8].max()
    return out


def round_one_tie():
    """The first round opens the block of the largest bound (510: two points meet a 255 cell at different leaves), whose best
    leaf scores 255. Blocks of bound exactly 255 hold leaves of the same score and a lower index: the second round must open
    a block whose bound equals the best leaf found."""
    hi = _grid(0.1, [[5, 0, 0], [-8, -3, 0]], [32767, 32767])
    hp = np.array([[0, 0, 0], [0, 0.2, 0]], f32)
    lo = _grid(0.5, np.zeros((1, 3)), [20000])
    c = _case("round_one_tie", hi, lo, hp, hp, IDENTITY, 0.1, 1.2, 0.0, 0.0)
    m = c.run()
    bounds = _block_bounds(c, m)
    top = bounds.max()
    ox, oy, oz = m.offset
    b = bounds[(oz + m.wz) // 8, (oy + m.wxy) // 8, (ox + m.wxy) // 8]
    best_sum = int(round((float(m.score) - 0.1) / float(ref.STEP) * 2))
    assert top == 510 and b < top - (top >> 3) and b == 255 == best_sum
    assert len(m.tied) >= 2
    return c


# ----------------------------------------------------------------------------------------------- the gate
def gate_rejects_in_block(k):
    """64 leaves of one block with distinct scores; the gate turns down the best k, the (k+1)-th passes."""
    xy = np.stack(np.meshgrid(np.arange(8), np.arange(8), indexing="ij"), -1).reshape(-1, 2)
    values = 32767 - 400 * np.arange(64)
    hi = _grid(0.1, np.concatenate([xy, np.zeros((64, 1), int)], 1), values)
    hp = np.zeros((1, 3), f32)
    order = np.argsort(-ref.LUT[values], kind="stable")
    passing = xy[order[k:]]
    lo = _grid(0.1, np.concatenate([passing, np.zeros((len(passing), 1), int)], 1), [32767] * len(passing))
    c = _case(f"gate_rejects_{k}_in_block", hi, lo, hp, hp, IDENTITY, 0.1, 0.8, 0.0, 0.5)
    m = c.run()
    assert len(m.rejected) == k and m.found and all(0 <= m.offset_of(i)[0] < 8 for i in m.rejected)
    return c


def gate_rejects_best_block():
    """Every leaf of the block of the largest bound fails the gate; a block of lower bound holds the answer."""
    xy = np.stack(np.meshgrid(np.arange(8), np.arange(8), indexing="ij"), -1).reshape(-1, 2)
    good = np.concatenate([xy, np.zeros((64, 1), int)], 1)
    weak = good + [-16, 0, 0]
    hi = _grid(0.1, np.concatenate([good, weak]), [32767] * 64 + [20000] * 64)
    hp = np.zeros((1, 3), f32)
    lo = _grid(0.1, weak, [32767] * 64)
    c = _case("gate_rejects_best_block", hi, lo, hp, hp, IDENTITY, 0.1, 1.6, 0.0, 0.5)
    m = c.run()
    assert len(m.rejected) == 64 and m.offset[0] < -8
    return c


# ----------------------------------------------------------------------------------------------- every cell value
def all_values():
    """Values 1..32 767 in a 32^3 cube around one point: every 8-bit value is a leaf score (value 5 462 sits on the .5 tie)."""
    cube = np.stack(np.meshgrid(*[np.arange(-16, 16)] * 3, indexing="ij"), -1).reshape(-1, 3)[1:, ::-1]   # (x, y, z), z slowest
    hi = _grid(0.1, cube, np.arange(1, 32768))
    hp = np.zeros((1, 3), f32)
    lo = _grid(0.5, np.zeros((1, 3)), [20000])
    c = _case("all_values", hi, lo, hp, hp, IDENTITY, 0.1, 1.6, 1.6, 0.0)
    m = c.run()
    leaf = m.scores[:32, :32, :32].reshape(-1)[1:]
    assert np.array_equal(leaf, ref.to_probability(ref.LUT[1:], 1))
    frac = ((ref.value_to_probability(5462) - ref.K_MIN) * (f32(255.0) / (ref.K_MAX - ref.K_MIN))).astype(np.float64)
    assert frac == 42.5 and ref.LUT[5462] == 43
    return c


# ----------------------------------------------------------------------------------------------- scenes
def scene(beams, k=0, min_score=0.15, min_low=0.3, seed=5):
    """A synthetic-scene submap (helpers.workload) at the stock 5 m x 5 m x 1 m window and pose-graph options, the node guess
    displaced by up to half the window."""
    import orc
    from helpers import workload
    w = workload(beams=beams, num_map_scans=20, num_scans=2)
    hi = ref.SparseGrid.from_export(w["hi"].resolution, w["hi"].export())
    lo = ref.SparseGrid.from_export(w["lo"].resolution, w["lo"].export())
    pts = orc.ingest_scan(w["opts"], w["scans"][k], w["origin"], w["prev"][k], w["truth"][k])["returns_tracking"]
    hk, _ = orc.adaptive_voxel_filter(pts, 2.0, 150, 15.0)
    lk, _ = orc.adaptive_voxel_filter(pts, 4.0, 200, 60.0)
    guess = np.array(w["truth"][k], np.float64)
    guess[:3] += np.random.default_rng(seed).uniform(-1, 1, 3) * [2.0, 2.0, 0.4]
    c = _case(f"scene{beams}_{k}_ms{min_score}", hi, lo, pts[hk], pts[lk], guess, min_score, 5.0, 1.0, min_low)
    assert ref.window(5.0, 1.0, hi.resolution) == (50, 10) and c.path == "pruned"
    return c


def _pick(generator, index):
    return lambda: generator()[index]


def _registry():
    r = {}
    for n_hi, n_lo in CLOUD_SIZES:
        r[f"cloud_hi{n_hi}_lo{n_lo}"] = functools.partial(cloud_size, n_hi, n_lo)
    for p in range(8):
        r[f"brick_rows_phase{p}"] = functools.partial(brick_rows, p)
    for g in (grid_edge_small, grid_edge_large, axis_8000, far_corners, margin_brick):
        r[{"grid_edge_small": "grid_edge_bits1", "grid_edge_large": "grid_edge_bits8"}.get(g.__name__, g.__name__)] = g
    for xy, z, want in WINDOWS:
        r[f"window_{want[0]}_{want[1]}"] = functools.partial(window_case, xy, z, want)
    for w in (399, 400):
        r[f"block_limit_{w}"] = functools.partial(block_limit, w)
    for res, k, side in WINDOW_TIES:
        r[f"window_tie_{res}_{k}_{side}"] = functools.partial(window_tie, res, k, side)
    r["all_leaves_0.1"], r["symmetric_ties"], r["tie_gate"] = all_leaves_equal, symmetric_ties, tie_gate
    r["at_min_score"], r["below_min_score"] = _pick(at_min_score, 0), _pick(at_min_score, 1)
    r["at_min_low"], r["above_min_low"] = _pick(at_min_low, 0), _pick(at_min_low, 1)
    r["round_one_tie"] = round_one_tie
    for k in (1, 2, 40):
        r[f"gate_rejects_{k}_in_block"] = functools.partial(gate_rejects_in_block, k)
    r["gate_rejects_best_block"], r["all_values"] = gate_rejects_best_block, all_values
    r["scene16_0_ms0.15"] = functools.partial(scene, 16, 0)
    r["scene16_1_ms0.55"] = functools.partial(scene, 16, 1, 0.55, 0.55)
    r["scene64_0_ms0.15"] = functools.partial(scene, 64, 0)
    return r


REGISTRY = _registry()
NAMES = list(REGISTRY)
NOT_SMALL = {"cloud_hi1023_lo64", "cloud_hi1024_lo64", "cloud_hi1025_lo64", "cloud_hi2049_lo64", "block_limit_399",
             "block_limit_400", "scene16_0_ms0.15", "scene16_1_ms0.55", "scene64_0_ms0.15"}
# data within 3 cells of -8 192: the reference's PrecomputeGrid grows its grid past the +-8 192 limit (CHECK failure)
NOT_IN_ORACLE = {"grid_edge_bits8"}


@functools.lru_cache(maxsize=None)
def get(name):
    c = REGISTRY[name]()
    assert c.name == name
    return c


def all_cases():
    return [get(n) for n in NAMES]
