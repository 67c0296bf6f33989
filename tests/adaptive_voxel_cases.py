"""Clouds on the edges of the device adaptive voxel filter (d-liom_b200/csrc/dl_voxel.cu), shared by the CPU oracle test and
the GPU test. Every generator checks with the numpy reference (adaptive_voxel_reference.py) that its cloud lands where its
name says: the cropped size, the voxel count or the cell box at the edge that decides the path, on the stated side of the
limit. A case is (name, rows, (max_length, min_num_points, max_range)).

The device limits the generators aim at:
  REGISTER_POINTS   8 192  cropped points the single-CTA search holds in registers (8 per thread)
  FAST_CAPACITY    22 528  cropped points of the fast mode: registers plus 14 336 in shared memory; above it, generic mode
  HASH_SLOTS        4 096  slots of the fast mode's shared hash table
  BYTE_MAP_CELLS   49 152  cells of the byte map that counts a pass when the cloud's cell box fits in it
  PACK_MIN, PACK_MAX       cells in [-2^20, 2^20 - 2] pack into a 63-bit key; any other cell sends the pair to generic mode
  ALWAYS_DIVIDES   ~1.04e6 quotients above it always take the exact division in round_div (dl_math.cuh)
"""
import collections

import numpy as np

import adaptive_voxel_reference as R

f32 = np.float32
REGISTER_POINTS = 8192
FAST_CAPACITY = 22528
HASH_SLOTS = 4096
BYTE_MAP_CELLS = 49152
PACK_MIN, PACK_MAX = -2 ** 20, 2 ** 20 - 2
# round_div's shortcut keeps x * (1 / edge) only when 0.5 - |distance to the nearest integer| > |q| * 4.8e-7: from this |q| on
# it never can, and every quotient takes the division
ALWAYS_DIVIDES = 0.5 / 4.8e-7
PADDED_ROWS = 8193  # padded() fills every cloud up to at least this many rows

Case = collections.namedtuple("Case", "name rows opts")


def side(value, limit):
    return int(np.sign(value - limit))


def outside_points(k, max_range, rng):
    """k points beyond max_range in random directions (1.5x to 4x the range)."""
    d = rng.normal(size=(k, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (d * rng.uniform(1.5, 4.0, (k, 1)) * max_range).astype(f32)


def interleave(inside, outside, rng):
    """Rows of `inside` in their order with the rows of `outside` scattered between them."""
    n = len(inside) + len(outside)
    mask = np.zeros(n, bool)
    mask[rng.choice(n, len(inside), replace=False)] = True
    out = np.empty((n, inside.shape[1]), f32)
    out[mask], out[~mask] = inside, outside
    return out


def padded(inside, max_range, rng, extra=500):
    """`inside` with out-of-range rows interleaved, at least PADDED_ROWS rows in all."""
    k = max(extra, PADDED_ROWS - len(inside))
    return interleave(np.asarray(inside, f32), outside_points(k, max_range, rng), rng)


def cropped(case):
    rows = R.xyz(case.rows)
    return rows[R.crop(rows, case.opts[2])]


def result_edge(case):
    return R.search(case.rows, *case.opts)[2]


# ------------------------------------------------------------------------------------------- cropped size around the storage
def storage_case(m, limit, expect):
    """m cropped points uniform in a 10 m cube (the first edge falls short: about 216 voxels of 2 m against 1 500), with a
    quarter as many out-of-range rows interleaved."""
    rng = np.random.RandomState(m)
    opts = (2.0, 1500.0, 20.0)
    inside = rng.uniform(-5, 5, (m, 3)).astype(f32)
    rows = interleave(inside, outside_points(m // 4, opts[2], rng), rng)
    case = Case(f"cropped_{m}", rows, opts)
    c = cropped(case)
    assert side(len(c), limit) == expect and len(rows) > len(c)
    assert R.num_voxels(c, opts[0]) < opts[1] < len(c)
    assert R.num_voxels(c, result_edge(case)) <= HASH_SLOTS
    return case


def storage_cases():
    return [storage_case(REGISTER_POINTS - 1, REGISTER_POINTS, -1), storage_case(REGISTER_POINTS, REGISTER_POINTS, 0),
            storage_case(REGISTER_POINTS + 1, REGISTER_POINTS, 1), storage_case(FAST_CAPACITY - 1, FAST_CAPACITY, -1),
            storage_case(FAST_CAPACITY, FAST_CAPACITY, 0), storage_case(FAST_CAPACITY + 1, FAST_CAPACITY, 1)]


# ------------------------------------------------------------------------------------------- sparse enough / first edge
def sparse_case(m, min_num_points, expect):
    """m cropped points against min_num_points: at or below it the cropped cloud is the result with no pass."""
    rng = np.random.RandomState(int(m * 10 + min_num_points))
    opts = (2.0, float(min_num_points), 15.0)
    case = Case(f"cropped_{m}_vs_min_{min_num_points:g}", padded(rng.uniform(-5, 5, (m, 3)), opts[2], rng), opts)
    assert side(len(cropped(case)), f32(min_num_points)) == expect
    return case


def first_edge_case(voxels, min_num_points, expect):
    """`voxels` occupied 2 m cells (60 points each, jittered inside the cell) against min_num_points."""
    rng = np.random.RandomState(voxels)
    opts = (2.0, float(min_num_points), 40.0)
    grid = np.stack(np.meshgrid(*[np.arange(-5, 5)] * 3, indexing="ij"), -1).reshape(-1, 3)
    centres = grid[rng.choice(len(grid), voxels, replace=False)] * 2.0
    pts = np.repeat(centres, 60, axis=0) + rng.uniform(-0.9, 0.9, (voxels * 60, 3))
    case = Case(f"voxels_{voxels}_at_max_length_vs_min_{min_num_points:g}", padded(pts[rng.permutation(len(pts))], opts[2], rng),
                opts)
    assert side(R.num_voxels(cropped(case), opts[0]), f32(min_num_points)) == expect
    return case


def threshold_cases():
    return [sparse_case(150, 150, 0), sparse_case(150 + 1, 150, 1), sparse_case(150, 150.5, -1), sparse_case(150 + 1, 150.5, 1),
            first_edge_case(150, 150, 0), first_edge_case(150 - 1, 150, -1), first_edge_case(151, 150.5, 1),
            first_edge_case(150, 150.5, -1)]


# ------------------------------------------------------------------------------------------- shared hash table at the result
def hash_case(voxels, expect):
    """Points at k * L/2 along x (k = 1 .. voxels - 1) and one at 1 000 * L/2 along y: at L pairs of them share a cell (k / 2 on a
    tie rounds away from zero), at L/2 every point has its own, and every refinement edge above L/2 merges some, so the result
    edge is L/2 with `voxels` voxels = min_num_points. The cell box there (voxels x 1 001 x 1) is far beyond the byte map."""
    rng = np.random.RandomState(voxels)
    opts = (0.5, float(voxels), 2000.0)
    pts = np.zeros((voxels, 3), f32)
    pts[:-1, 0] = np.arange(1, voxels) * f32(0.25)
    pts[-1, 1] = 1000 * f32(0.25)
    pts = np.tile(pts, (2, 1))[rng.permutation(2 * voxels)]     # twice each: more points than min_num_points
    case = Case(f"hash_{voxels}_voxels_at_result_edge", padded(pts, opts[2], rng), opts)
    edge = result_edge(case)
    c = cropped(case)
    assert edge == f32(0.25) and side(R.num_voxels(c, edge), HASH_SLOTS) == expect
    assert np.prod(R.cell_box(c, edge)) > BYTE_MAP_CELLS
    assert R.search(case.rows, *opts)[1][-1] != edge         # the last pass was a refinement: the result is rebuilt
    return case


def many_voxels_case(voxels):
    """`voxels` occupied 1 m cells of a 32 x 16 x 17 block, three points each; the first edge suffices, with far more voxels
    than the search's result table holds (generic mode)."""
    rng = np.random.RandomState(voxels)
    opts = (1.0, 150.0, 100.0)
    grid = np.stack(np.meshgrid(np.arange(32), np.arange(16), np.arange(17), indexing="ij"), -1).reshape(-1, 3)
    centres = grid[rng.choice(len(grid), voxels, replace=False)].astype(f32)
    pts = np.repeat(centres, 3, axis=0) + rng.uniform(-0.45, 0.45, (3 * voxels, 3))
    case = Case(f"voxels_{voxels}_at_max_length", padded(pts[rng.permutation(len(pts))], opts[2], rng), opts)
    n = R.num_voxels(cropped(case), opts[0])
    assert n == voxels and n >= opts[1]
    return case


def table_cases():
    return [hash_case(HASH_SLOTS, 0), hash_case(HASH_SLOTS + 1, 1), many_voxels_case(8192), many_voxels_case(8193)]


# ------------------------------------------------------------------------------------------- byte-map box
def box_case(name, box, expect, pairs=1000):
    """Sites on the L/2 = 0.25 m lattice inside the cell box `box` (its two corners occupied) in pairs k, k + x with odd k.x: at
    L the pair shares a cell (tie away from zero), at L/2 it does not, and the refinement edges above L/2 merge some pairs, so
    the search ends at L/2 with min_num_points = its voxel count. The box there is `box` cells."""
    rng = np.random.RandomState(sum(box))
    lat = np.stack([rng.randint(0, (box[0] - 1) // 2, pairs) * 2 + 1] + [rng.randint(0, b, pairs) for b in box[1:]], 1)
    sites = np.concatenate([[[0, 0, 0], [box[0] - 1, box[1] - 1, box[2] - 1]], lat, lat + [1, 0, 0]])
    pts = sites.astype(f32) * f32(0.25)
    n = R.num_voxels(pts, 0.25)
    opts = (0.5, float(n), 20000.0)
    case = Case(name, padded(pts[rng.permutation(len(pts))], opts[2], rng), opts)
    k, passes, edge = R.search(case.rows, *opts)
    assert edge == f32(0.25) and passes[-1] != edge and n <= HASH_SLOTS
    assert R.cell_box(cropped(case), edge) == tuple(box) and side(int(np.prod(box)), BYTE_MAP_CELLS) == expect
    return case


def box_cases():
    return [box_case("box_48x32x32_cells", (48, 32, 32), 0), box_case("box_49x32x32_cells", (48 + 1, 32, 32), 1),
            box_case("box_49152x1x1_cells", (BYTE_MAP_CELLS, 1, 1), 0),
            box_case("box_49153x1x1_cells", (BYTE_MAP_CELLS + 1, 1, 1), 1)]


# ------------------------------------------------------------------------------------------- key packing
def packing_case(cell, bound, expect):
    """Three points with `cell` on one axis each (edge 2^-10 m, exact), 300 ordinary points near the origin; the first edge
    suffices. `expect` is the side of `cell` against the packable bound."""
    rng = np.random.RandomState(abs(cell) % 1000)
    edge = 2.0 ** -10
    opts = (edge, 50.0, 4096.0)
    far = np.eye(3, dtype=np.float64) * cell * edge
    pts = np.concatenate([rng.uniform(-1, 1, (300, 3)), far]).astype(f32)
    case = Case(f"key_cell_{cell}", padded(pts[rng.permutation(len(pts))], opts[2], rng), opts)
    cc = R.cells(cropped(case), edge)
    extreme = cc.min() if bound == PACK_MIN else cc.max()
    assert extreme == cell and side(extreme, bound) == expect and R.search(case.rows, *opts)[2] == f32(edge)
    return case


def packing_after_halving_case():
    """Cells at +-2^19 at the first edge pack; the first edge falls short, and at L/2 the cell 2^20 does not: the fast mode
    gives up in the middle of the search and generic mode redoes it. Every edge keeps the same voxels: 8 passes."""
    rng = np.random.RandomState(19)
    edge = 2.0 ** -10
    pts = np.concatenate([rng.uniform(-0.5, 0.5, (200, 3)), np.eye(3) * 2 ** 19 * edge, -np.eye(3) * 2 ** 19 * edge]).astype(f32)
    pts = np.tile(pts, (6, 1))                                  # 1 236 points in 206 voxels at every edge
    opts = (edge, 1000.0, 4096.0)
    case = Case("key_cell_2^19_packs_only_at_the_first_edge", padded(pts, opts[2], rng), opts)
    cc = R.cells(cropped(case), edge)
    assert cc.max() == 2 ** 19 <= PACK_MAX < 2 * cc.max() and len(R.search(case.rows, *opts)[1]) == 8
    return case


def packing_cases():
    return [packing_case(PACK_MIN, PACK_MIN, 0), packing_case(PACK_MAX, PACK_MAX, 0), packing_case(PACK_MIN - 1, PACK_MIN, -1),
            packing_case(PACK_MAX + 1, PACK_MAX, 1), packing_after_halving_case()]


# ------------------------------------------------------------------------------------------- rounding
def near_ties(k, edge, rng):
    """float32 (k + 1/2) * edge moved by -4 .. 4 ulps, per coordinate."""
    x = ((np.asarray(k, np.float64) + 0.5) * np.float64(f32(edge))).astype(f32)
    u = rng.randint(-4, 5, x.shape)
    while (u != 0).any():
        x = np.where(u > 0, np.nextafter(x, f32(np.inf)), np.where(u < 0, np.nextafter(x, f32(-np.inf)), x)).astype(f32)
        u -= np.sign(u)
    return x


def rounding_case(j, max_length=1.5):
    """3 000 points on near-ties of the edge e = max_length / 2^j, |k| <= 8 per axis; min_num_points = the voxel count at e, so
    the pass at e decides the search (the coarser edges of the halving sequence hold fewer voxels)."""
    rng = np.random.RandomState(100 + j)
    e = f32(max_length) / f32(2 ** j)
    pts = near_ties(rng.randint(-8, 9, (3000, 3)), e, rng)
    n = R.num_voxels(pts, e)
    opts = (max_length, float(n), 100.0)
    case = Case(f"near_ties_of_edge_max_length/2^{j}", padded(pts, opts[2], rng), opts)
    k, passes, edge = R.search(case.rows, *opts)
    assert e in passes and all(R.num_voxels(pts, f32(max_length) / f32(2 ** i)) < n for i in range(j))
    return case


def rounding_far_case(k0, name, generic):
    """Near-ties at the first edge with quotients from k0 on the x axis: where the reciprocal shortcut always takes the division
    (|q| > 2^20) and still packs, or beyond 2^22 (division in every path, key not packable)."""
    rng = np.random.RandomState(k0 % 997)
    e = f32(1.5)
    kx = k0 + rng.randint(0, 60, 2000)
    pts = np.stack([near_ties(kx, e, rng), near_ties(rng.randint(-8, 9, 2000), e, rng),
                    near_ties(rng.randint(-8, 9, 2000), e, rng)], 1)
    n = R.num_voxels(pts, e)
    opts = (float(e), float(n), 1.5 * (k0 + 100) * 1.5)
    case = Case(name, padded(pts, opts[2], rng), opts)
    cc = R.cells(cropped(case), e)
    assert R.search(case.rows, *opts)[2] == e and (cc.max() > PACK_MAX) == generic and cc[:, 0].min() > ALWAYS_DIVIDES
    return case


def rounding_cases():
    return [rounding_case(j) for j in range(8)] + [rounding_far_case(2 ** 20 - 70, "near_ties_quotient_2^20_packable", False),
                                                   rounding_far_case(2 ** 22 + 8, "near_ties_quotient_2^22_generic", True)]


# ------------------------------------------------------------------------------------------- exhausted search, input order
def exhausted_case():
    """9 000 copies of one point: every edge has one voxel, the halving runs out after L/128 and the result is that pass."""
    rng = np.random.RandomState(9)
    opts = (2.0, 150.0, 15.0)
    case = Case("one_voxel_exhausts_the_search", padded(np.tile([[1.0, -2.0, 0.5]], (9000, 1)), opts[2], rng), opts)
    keep, passes, edge = R.search(case.rows, *opts)
    assert len(passes) == 8 and edge == passes[-1] == f32(2.0) / 128 and len(keep) == 1
    return case


def order_case():
    """20 000 cropped points in 2 000 voxels of 1 m, members in random order (about 10 per voxel, spread over the 1 024-id rounds
    and both sides of the register / shared-memory split), and one voxel whose members sit at ids 1 023, 1 024, 8 191, 8 192,
    8 193, 9 000 and 19 999 with the lowest id last in no round."""
    rng = np.random.RandomState(20)
    m = 20000
    grid = np.stack(np.meshgrid(*[np.arange(-7, 7)] * 3, indexing="ij"), -1).reshape(-1, 3)
    centres = grid[rng.choice(len(grid), 2000, replace=False)].astype(f32)
    owner = rng.randint(1, 2000, m)
    special = [1023, 1024, 8191, 8192, 8193, 9000, 19999]
    owner[special] = 0
    owner[(owner == 0) & ~np.isin(np.arange(m), special)] = 1
    pts = centres[owner] + rng.uniform(-0.45, 0.45, (m, 3)).astype(f32)
    opts = (1.0, 150.0, 40.0)
    case = Case("voxels_split_over_rounds_and_storage", interleave(pts.astype(f32), outside_points(3000, opts[2], rng), rng), opts)
    c = cropped(case)
    keep = R.voxel_filter(c, 1.0)
    assert len(c) == m and 1023 in keep and not np.isin(special[1:], keep).any() and len(keep) <= HASH_SLOTS
    assert REGISTER_POINTS < m <= FAST_CAPACITY and R.search(case.rows, *opts)[2] == f32(1.0)
    return case


def street_cases(orc):
    """The returns of a 16-beam street sweep (first voxel filter 5 cm: 18 000 returns) in random order, under the two filters of
    the front end."""
    from helpers import workload
    w = workload()
    opts = orc.FrontEndOptions.defaults(voxel_filter_size=0.05)
    pts = orc.ingest_scan(opts, w["scans"][0], w["origin"], w["prev"][0], w["cur"][0])["returns_tracking"]
    pts = pts[np.random.RandomState(3).permutation(len(pts))]
    return [Case("shuffled_street_scan_high_resolution", pts, (2.0, 150.0, 15.0)),
            Case("shuffled_street_scan_low_resolution", pts, (4.0, 200.0, 60.0))]


# ------------------------------------------------------------------------------------------- row formats, special values
def format_cases():
    """Strides 3, 4 and 8 with NaN in the unused columns; NaN and infinite rows (cropped away); a point exactly at max_range
    (5, 12, 0) at 13 m and one a float above it; clouds of 0, 1 and 8 193 rows."""
    rng = np.random.RandomState(48)
    opts = (1.0, 400.0, 13.0)
    pts = rng.uniform(-7, 7, (9000, 3)).astype(f32)
    pts[::97] = np.nan
    pts[5::211, 1] = np.inf
    pts[3] = [5, 12, 0]
    pts[4] = [5, np.nextafter(f32(12), f32(13)), 0]
    r = R.norms(pts)
    assert r[3] == f32(13) and r[4] > f32(13)
    c = R.crop(pts, opts[2])
    assert 3 in c and 4 not in c and not np.isin(np.arange(0, 9000, 97), c).any()
    out = []
    for stride in (3, 4, 8):
        rows = np.full((len(pts), stride), np.nan, f32)
        rows[:, :3] = pts
        out.append(Case(f"stride_{stride}_nan_rows_point_at_max_range", rows, opts))
    for n in (0, 1, PADDED_ROWS):
        out.append(Case(f"rows_{n}", rng.uniform(-5, 5, (n, 3)).astype(f32), (2.0, 150.0, 15.0)))
    return out


def all_cases(orc=None):
    cases = (storage_cases() + threshold_cases() + table_cases() + box_cases() + packing_cases() + rounding_cases() +
             [exhausted_case(), order_case()] + format_cases())
    if orc is not None:
        cases += street_cases(orc)
    return cases

