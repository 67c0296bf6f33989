"""Inputs for the range-data inserter, one generator per edge of RangeDataInserter3D::Insert and the grid it writes.

Every generator returns a Case and checks, with the numpy reference, that its input really sits on the side of the edge it
is named for; a reader can see the edge in the assertion at its end. A case is a list of Inserts into one grid, run in
order; `status` is what the reference reports for each (0, or the status of the CHECK the reference fails).
"""
from dataclasses import dataclass, field

import numpy as np

import range_data_inserter_reference as ref

f32 = np.float32


@dataclass
class Step:
    origin: np.ndarray
    returns: np.ndarray
    hit: float = 0.55
    miss: float = 0.49
    num_free: int = 2


@dataclass
class Case:
    name: str
    resolution: float
    steps: list
    status: list = field(default_factory=list)

    def run_reference(self):
        """-> (grid after every step that succeeded, statuses); a failing step leaves the grid as it was."""
        g = ref.Grid(self.resolution)
        statuses = []
        for s in self.steps:
            try:
                ref.insert(g, s.origin, s.returns, s.hit, s.miss, s.num_free)
                statuses.append(0)
            except ref.InsertError as e:
                statuses.append(e.status)
        return g, statuses


def _case(name, resolution, steps):
    c = Case(name, resolution, steps)
    c.status = c.run_reference()[1]
    return c


def _rays(step, resolution):
    return ref.rays(step.origin, step.returns, resolution, step.num_free)


def _p(*rows):
    return np.array(rows, f32).reshape(-1, 3)


# ----------------------------------------------------------------------------------------------- generators
def reference_fixture():
    """range_data_inserter_3d_test.cc: hit 0.7, miss 0.4, 1000 free-space voxels, forty Inserts of four rays."""
    step = Step(_p(0, 0, -4), _p([-3, -1, 4], [-2, 0, 4], [-1, 1, 4], [0, 2, 4]), 0.7, 0.4, 1000)
    hits, misses, _, ns = _rays(step, 1.0)
    assert (ns < step.num_free).all() and (misses == [0, 0, -4]).all(axis=1).any()   # whole rays, origin cell included
    return _case("reference_fixture", 1.0, [step] * 40)


def directions():
    """Every delta with components in -3..3 from an origin cell: 26 directions, num_samples 0..3, mixed signs."""
    d = np.stack(np.meshgrid(*[np.arange(-3, 4)] * 3, indexing="ij"), axis=-1).reshape(-1, 3)
    origin = _p(0.3, -0.2, 0.4)
    steps = [Step(origin, (d + _p(0.1, -0.3, 0.2)).astype(f32), num_free=nf) for nf in (2, 3)]
    hits, misses, ray, ns = _rays(steps[1], 1.0)
    delta = hits[ray] - [0, 0, 0]
    pos = np.concatenate([np.arange(n - min(n, 3), n) for n in ns])
    floor = np.floor_divide(delta * pos[:, None], np.maximum(ns[ray], 1)[:, None])
    assert set(ns.tolist()) == {0, 1, 2, 3}
    assert len({tuple(np.sign(x)) for x in d if x.any()}) == 26
    assert (misses != floor).any()                                    # truncation and floor part ways on some sample
    return _case("directions", 1.0, steps)


def num_free_edges():
    """num_free of 0, 1, 2, num_samples - 1, num_samples and 8192 on rays of 7 samples, and a hit in the origin cell."""
    origin = _p(-0.2, 0.1, 0.3)
    returns = _p([7, 3, -2], [-7, 1, 5], [2, -7, -7], [0, 0, 7], [7, -7, 1], [0, 0, 0.4])
    cases = []
    for nf in (0, 1, 2, 6, 7, 8192):
        step = Step(origin, returns, num_free=nf)
        hits, misses, _, ns = _rays(step, 1.0)
        origin_is_miss = (misses == [0, 0, 0]).all(axis=1).any()
        assert set(ns.tolist()) == {0, 7}                               # a hit in the origin cell too
        assert len(misses) == np.minimum(ns, nf).sum()
        assert origin_is_miss == (nf >= 7)                            # the origin cell takes a miss iff nf >= num_samples
        cases.append(_case(f"num_free_{nf}", 1.0, [step]))
    return cases


def one_cell_many_returns():
    """10 000 returns in one cell: one hit update, one update per miss cell."""
    rng = np.random.RandomState(7)
    returns = (_p(12, -5, 3) + rng.uniform(-0.45, 0.45, (10000, 3))).astype(f32)
    step = Step(_p(0, 0, 0), returns, num_free=4)
    hits, misses, _, _ = _rays(step, 1.0)
    assert len(np.unique(hits, axis=0)) == 1 and len(returns) == 10000
    return _case("one_cell_many_returns", 1.0, [step, step])


def shared_word():
    """Neighbouring x cells 2k (a hit) and 2k + 1 (a miss) share one 32-bit word of the brick; so do 2k (a miss) and 2k + 1
    (a hit)."""
    origin = _p(11.2, 0.1, 0.0)
    returns = _p([10, 0, 0], [13, 0, 0], [13, 2, 1], [8, 4, -1], [-20, 3, 2], [-21, 3, 2])
    step = Step(origin, returns, num_free=3)
    hits, misses, _, _ = _rays(step, 1.0)
    hk, mk = np.unique(ref.order_key(hits)), np.setdiff1d(ref.order_key(misses), ref.order_key(hits))
    # the key's lowest bit is the x parity inside the brick: keys k and k ^ 1 are the two halves of one word
    assert np.intersect1d(hk[hk % 2 == 0], mk[mk % 2 == 1] - 1).size > 0      # hit low half, miss high half
    assert np.intersect1d(hk[hk % 2 == 1] - 1, mk[mk % 2 == 0]).size > 0      # miss low half, hit high half
    return _case("shared_word", 1.0, [step, step])


def hit_beats_miss():
    """The hit cell of ray A is a miss cell of ray B: it takes the hit table once, never the miss table."""
    step = Step(_p(0, 0, 0), _p([3, 0, 0], [4, 0, 0], [5, 1, 0], [2, 0, 0]), num_free=3)
    hits, misses, _, _ = _rays(step, 1.0)
    assert np.intersect1d(ref.order_key(hits), ref.order_key(misses)).size >= 2
    return _case("hit_beats_miss", 1.0, [step, step])


def _straddle(k, res):
    """The adjacent float32 values (a, b), b = nextafter(a, +inf), near (k + 1/2) * res whose cell indices differ: the
    rounding boundary of lround(float(x / res))."""
    x = f32((k + 0.5) * float(res))
    for _ in range(64):
        x = np.nextafter(x, f32(-np.inf))
    for _ in range(128):
        y = np.nextafter(x, f32(np.inf))
        if ref.cell_index(np.array([[x, 0, 0]], f32), res)[0, 0] != ref.cell_index(np.array([[y, 0, 0]], f32), res)[0, 0]:
            return x, y
        x = y
    raise AssertionError(f"no boundary near ({k} + 1/2) * {res}")


def half_ulp(resolution):
    """Points one ulp either side of each rounding boundary (k + 1/2) * resolution, as hit cells and as the origin cell."""
    res = f32(resolution)
    bounds = [_straddle(k, res) for k in (-40, -7, -3, -1, 0, 1, 2, 5, 33)]
    below = np.array([a for a, _ in bounds], f32)
    above = np.array([b for _, b in bounds], f32)
    assert (ref.cell_index(np.stack([below] * 3, 1), res) != ref.cell_index(np.stack([above] * 3, 1), res)).all()
    pts = np.concatenate([below, above])
    grid = np.stack(np.meshgrid(pts, pts[::5], indexing="ij"), axis=-1).reshape(-1, 2)
    returns = np.concatenate([grid, np.full((len(grid), 1), above[5], f32)], axis=1).astype(f32)
    cases = []
    for side, o in (("below", below[4]), ("above", above[4])):   # the origin on either side of the boundary at k = 0
        cases.append(_case(f"half_ulp_{resolution}_{side}", resolution, [Step(np.array([o, o, o], f32), returns, num_free=3)]))
    return cases


def range_limits():
    """Cells -8192 and 8191 pass; 8192 and -8193 fail; growth from bits 1 to 8 in one Insert; a miss outside fails."""
    o = _p(0.2, 0.3, -0.1)
    edge = _p([-8192, 0, 0], [8191, 0, 0], [0, -8192, 0], [0, 8191, 0], [0, 0, -8192], [0, 0, 8191])
    ok = Step(o, edge)
    hits, misses, _, _ = _rays(ok, 1.0)
    assert ref.in_range(np.concatenate([hits, misses])) and ref.bits_for(hits) == 8     # bits 1 -> 8 in one Insert
    high, low = Step(o, _p([8192, 0, 0])), Step(o, _p([0, -8193, 0]))
    far = Step(_p(-9000, 0, 0), _p([-8190, 0, 0]), num_free=1000)    # hit inside, misses outside
    h, m, _, _ = _rays(far, 1.0)
    assert ref.in_range(h) and not ref.in_range(m)
    cases = [_case("limits_pass", 1.0, [ok]), _case("limit_8192", 1.0, [ok, high, Step(o, _p([1, 2, 3]))]),
             _case("limit_-8193", 1.0, [low, ok]), _case("limit_miss_outside", 1.0, [Step(o, _p([5, 5, 5])), far, ok])]
    assert [c.status for c in cases] == [[0], [0, ref.ERR_GRID_RANGE, 0], [ref.ERR_GRID_RANGE, 0],
                                         [0, ref.ERR_GRID_RANGE, 0]]
    return cases


def origin_beyond_range():
    """The origin 9 000 cells out, every touched cell inside +-8192: the reference inserts without trouble."""
    step = Step(_p(-9000, 0.3, 0.2), _p([-8000, 1, 0], [-8001, -2, 3], [-7990, 0, 0]))
    hits, misses, _, _ = _rays(step, 1.0)
    assert not ref.in_range(ref.cell_index(step.origin, 1.0)) and ref.in_range(np.concatenate([hits, misses]))
    return _case("origin_beyond_range", 1.0, [step, Step(_p(0, 0, 0), _p([3, 2, 1]))])


def num_samples_limit():
    """Rays of 32 767 samples pass, of 32 768 samples are refused before the grid changes (CHECK_LT(num_samples, 1 << 15))."""
    hit = _p([8191, 5, -3])
    passing = Step(_p(8191 - 32767, 5, -3), hit)
    passing_wide = Step(_p(8191 - 32767, 5, -3), hit, num_free=8192)
    refused = Step(_p(8191 - 32768, 5, -3), np.concatenate([hit, _p([0, 0, 0])]))
    assert _rays(passing, 1.0)[3].max() == 32767 and _rays(refused, 1.0)[3].max() == 32768
    cases = [_case("num_samples_32767", 1.0, [passing, passing_wide]),
             _case("num_samples_32768", 1.0, [Step(_p(0, 0, 0), _p([1, 1, 1])), refused, passing])]
    assert cases[0].status == [0, 0] and cases[1].status == [0, ref.ERR_ARG, 0]
    return cases


def street(beams, resolution, scans=3):
    """Sweeps of the synthetic street scene, each inserted from its sensor origin in the scene frame."""
    import synth
    scene = synth.Scene(42)
    steps = []
    for k in range(scans):
        t = 2.0 + 0.1 * k
        rows = synth.make_scan(scene, beams, t)
        pose = synth.pose7(t)
        pts = np.stack([rows["x"], rows["y"], rows["z"]], axis=1).astype(np.float64)
        world = ref.rotate(pose[3:], pts) + pose[:3]
        steps.append(Step(pose[:3].astype(f32), world.astype(f32)))
    hits, misses, ray, ns = _rays(steps[0], resolution)
    assert len(hits) > 1000 * beams // 16 and ns.max() < ref.MAX_SAMPLES
    return _case(f"street_{beams}_{resolution}", resolution, steps)


def all_cases():
    cases = [reference_fixture(), directions(), *num_free_edges(), one_cell_many_returns(), shared_word(), hit_beats_miss()]
    for r in (0.05, 0.1, 0.3, 0.45, 1.0):
        cases += half_ulp(r)
    cases += range_limits() + [origin_beyond_range()] + num_samples_limit()
    for beams in (16, 64):
        for r in (0.1, 0.45):
            cases.append(street(beams, r))
    return cases
