"""The device grid write side (dl_grid_insert_range_data, dl_submap_insert_range_data and the batched builder's insert) against
the numpy reference of tests/range_data_inserter_reference.py, bit for bit: every cell, in iterator order, the number of
bricks in use, and the status of every call the reference refuses."""
import numpy as np
import pytest

import range_data_inserter_cases as cases
import range_data_inserter_reference as ref

pytestmark = pytest.mark.gpu

f32 = np.float32
ALL = cases.all_cases()
ODDS_PAIRS = [(0.55, 0.49), (0.7, 0.4), (0.9, 0.1), (0.99, 0.01), (0.5000001, 0.4999999), (0.50000001, 0.0)]


@pytest.fixture(scope="module")
def ctx():
    import dliom
    c = dliom.Context(0)
    yield c
    c.close()


def assert_same(device, reference):
    # the brick count first: an export brings the grid's host mirror up to date
    assert device.num_bricks == reference.num_bricks
    got, want = device.export(), reference.export()
    for a, b in zip(got, want):
        assert a.dtype == b.dtype and np.array_equal(a, b)


def device_insert(g, step):
    """-> the library's status of one Insert (0 on success)."""
    import dliom
    try:
        g.insert_range_data(step.origin, step.returns, step.hit, step.miss, step.num_free)
        return 0
    except dliom.DlError as e:
        return e.status


@pytest.mark.parametrize("case", ALL, ids=[c.name for c in ALL])
def test_case_equals_reference(ctx, case):
    """Every Insert of the case: the same cells, order, values and brick count as the reference, the same status; a refused
    Insert leaves the grid's cells as they were, and the next Insert still matches."""
    g, r = ctx.grid(case.resolution), ref.Grid(case.resolution)
    for step, status in zip(case.steps, case.status):
        before = g.export()
        assert device_insert(g, step) == status
        if status:
            for a, b in zip(g.export(), before):
                assert np.array_equal(a, b)
        else:
            ref.insert(r, step.origin, step.returns, step.hit, step.miss, step.num_free)
        assert_same(g, r)


# ----------------------------------------------------------------------------------------------- the odds tables, every entry
@pytest.mark.parametrize("hit,miss", ODDS_PAIRS)
def test_hit_table_every_entry(ctx, hit, miss):
    """Values 1..32767 in 32767 cells, one return at each cell centre with no free space: each cell takes hit_table[value].
    One more return in a fresh cell takes hit_table[0]."""
    idx = np.arange(32767)
    cells = np.stack([idx % 32, (idx // 32) % 32, idx // 1024], axis=1) - 16
    values = (idx + 1).astype(np.uint16)
    g, r = ctx.grid(1.0), ref.Grid(1.0)
    g.set_cells(cells[:, 0], cells[:, 1], cells[:, 2], values)
    r.set_cells(cells[:, 0], cells[:, 1], cells[:, 2], values)
    returns = np.concatenate([cells, [[40, 40, 40]]]).astype(f32)
    g.insert_range_data(np.zeros(3, f32), returns, hit, miss, 0)
    ref.insert(r, np.zeros(3, f32), returns, hit, miss, 0)
    assert_same(g, r)
    table = ref.tables(hit, miss)[0].astype(np.int64) - ref.UPDATE_MARKER
    got = g.lookup(np.concatenate([cells, [[40, 40, 40]]]))
    assert np.array_equal(got[:-1], table[1:]) and got[-1] == table[0]


@pytest.mark.parametrize("hit,miss", ODDS_PAIRS)
def test_miss_table_every_entry(ctx, hit, miss):
    """Cells along the six axes and four diagonals from the origin preset with values 1..32767 (the origin cell left at 0);
    one return at the far end of each direction with 8192 free-space voxels: every ray cell takes miss_table[value]."""
    ends = np.array([[8191, 0, 0], [-8192, 0, 0], [0, 8191, 0], [0, -8192, 0], [0, 0, 8191], [0, 0, -8192],
                     [3000, 3000, 3000], [-3000, 2999, -1], [2000, -4000, 1000], [-5, -6000, 6000]], f32)
    origin = np.array([0.2, -0.3, 0.1], f32)
    hits, misses, _, ns = ref.rays(origin, ends, 1.0, 8192)
    assert (ns <= 8192).all()                                     # every sample of every ray is a miss, the origin cell too
    keys = np.setdiff1d(np.unique(ref.order_key(misses)), ref.order_key(hits))
    keys = keys[keys != ref.order_key(np.zeros((1, 3), np.int64))[0]]
    assert len(keys) >= 32767
    preset = ref.key_to_cells(keys)
    values = (np.arange(len(keys)) % 32767 + 1).astype(np.uint16)
    g, r = ctx.grid(1.0), ref.Grid(1.0)
    g.set_cells(preset[:, 0], preset[:, 1], preset[:, 2], values)
    r.set_cells(preset[:, 0], preset[:, 1], preset[:, 2], values)
    g.insert_range_data(origin, ends, hit, miss, 8192)
    ref.insert(r, origin, ends, hit, miss, 8192)
    assert_same(g, r)
    table = ref.tables(hit, miss)[1].astype(np.int64) - ref.UPDATE_MARKER
    assert np.array_equal(g.lookup(preset), table[values]) and g.lookup(np.zeros((1, 3), np.int32))[0] == table[0]


# ----------------------------------------------------------------------------------------------- grid state between Inserts
def test_uploaded_grid_then_inserts_and_set_cells(ctx):
    """A grid uploaded from a reference-built one, its bricks allocated in an order that is not the iterator's, then device
    Inserts alternating three times with dl_grid_set_cells."""
    case = cases.street(16, 0.45, scans=4)
    built, _ = cases.Case("built", 0.45, case.steps[:2]).run_reference()
    x, y, z, v = built.export()
    order = np.random.RandomState(3).permutation(len(x))             # bricks allocated in shuffled order
    g, r = ctx.grid(0.45), ref.Grid(0.45)
    g.set_cells(x[order], y[order], z[order], v[order])
    r.set_cells(x[order], y[order], z[order], v[order])
    assert_same(g, r)
    rng = np.random.RandomState(5)
    for k, step in enumerate(case.steps[2:] + case.steps[:1]):
        g.insert_range_data(step.origin, step.returns, step.hit, step.miss, step.num_free)
        ref.insert(r, step.origin, step.returns, step.hit, step.miss, step.num_free)
        assert_same(g, r)
        cx, cy, cz, _ = r.export()
        pick = rng.choice(len(cx), 500, replace=False)
        new = rng.randint(1, 32768, 500).astype(np.uint16)
        fresh = np.array([[300 + k, -200, 7]])                    # and one cell in a brick of its own
        sx, sy, sz = (np.concatenate([a[pick], fresh[:, i]]) for i, a in enumerate((cx, cy, cz)))
        sv = np.concatenate([new, [1234]]).astype(np.uint16)
        g.set_cells(sx, sy, sz, sv)
        r.set_cells(sx, sy, sz, sv)
        assert_same(g, r)


# ----------------------------------------------------------------------------------------------- Submap3D::InsertRangeData
def _unit(q):
    q = np.asarray(q, np.float64)
    return q / np.linalg.norm(q)


POSES = {"identity": np.array([0, 0, 0, 1, 0, 0, 0.0]),
         "yaw": np.array([-412.0, 318.5, 2.25, *_unit([0.8, 0, 0, 0.6])]),
         "tilted": np.array([250.125, -733.75, -41.5, *_unit([0.7, 0.2, -0.3, 0.62])])}


def _street_local(pose, scans=2):
    """Street sweeps placed in the local frame around the submap's origin."""
    steps = cases.street(16, 0.1, scans=scans).steps
    return [((s.returns.astype(np.float64) + pose[:3]).astype(f32), (s.origin + pose[:3]).astype(f32)) for s in steps]


def submap_pair(ctx, hi_res=0.1, lo_res=0.45):
    return ctx.grid(hi_res), ctx.grid(lo_res), ref.Grid(hi_res), ref.Grid(lo_res)


@pytest.mark.parametrize("pose", list(POSES))
@pytest.mark.parametrize("max_range", [0, 1, 20])
def test_submap_insert_at_poses(ctx, pose, max_range):
    p = POSES[pose]
    dhi, dlo, rhi, rlo = submap_pair(ctx)
    for returns, origin in _street_local(p):
        ctx.submap_insert_range_data(dhi, dlo, p, origin, returns, max_range)
        _, near, _ = ref.submap_insert(rhi, rlo, p, origin, returns, max_range)
        if max_range == 0:
            assert len(near) == 0                                  # the high-resolution job drops out on the device count
    assert_same(dhi, rhi)
    assert_same(dlo, rlo)


def test_submap_insert_at_max_range_boundary(ctx):
    """Points whose submap-frame distance from the origin is exactly high_resolution_max_range after the float transform,
    and one ulp either side."""
    p = POSES["tilted"]
    t, q = ref.to_submap_transform(p)
    origin = (p[:3] + [0.25, -0.5, 0.125]).astype(f32)
    o = ref.transform(origin[None], t, q)[0]
    rng = np.random.RandomState(11)
    dirs = rng.normal(size=(4000, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    R = 20
    scale = np.linspace(1 - 8e-7, 1 + 8e-7, 17)
    local = (origin.astype(np.float64) + (dirs[:, None, :] * (R * scale)[None, :, None]).reshape(-1, 3)).astype(f32)
    sub = ref.transform(local, t, q)
    d = sub - o
    dist = np.sqrt(d[:, 0] * d[:, 0] + (d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]))
    R32 = f32(R)
    assert (dist == R32).sum() > 0
    assert (dist == np.nextafter(R32, f32(0))).sum() > 0 and (dist == np.nextafter(R32, f32(np.inf))).sum() > 0
    keep = (np.abs(dist - R32) <= 2 * (np.nextafter(R32, f32(np.inf)) - R32))
    returns = local[keep]
    dhi, dlo, rhi, rlo = submap_pair(ctx)
    ctx.submap_insert_range_data(dhi, dlo, p, origin, returns, R)
    _, near, _ = ref.submap_insert(rhi, rlo, p, origin, returns, R)
    assert 0 < len(near) < len(returns)
    assert_same(dhi, rhi)
    assert_same(dlo, rlo)


def test_submap_insert_all_beyond_range_and_empty(ctx):
    p = POSES["yaw"]
    dhi, dlo, rhi, rlo = submap_pair(ctx)
    (returns, origin), = _street_local(p, scans=1)
    far = (returns.astype(np.float64) + [0, 0, 50.0]).astype(f32)   # every point more than 20 m from the origin
    ctx.submap_insert_range_data(dhi, dlo, p, origin, far, 20)
    _, near, _ = ref.submap_insert(rhi, rlo, p, origin, far, 20)
    assert len(near) == 0 and len(dhi.export()[0]) == 0 and dhi.num_bricks == 0
    assert_same(dlo, rlo)
    ctx.submap_insert_range_data(dhi, dlo, p, origin, np.zeros((0, 3), f32), 20)
    assert_same(dhi, rhi)
    assert_same(dlo, rlo)
    ctx.submap_insert_range_data(dhi, dlo, p, origin, returns, 20)    # and a normal Insert after both
    ref.submap_insert(rhi, rlo, p, origin, returns, 20)
    assert_same(dhi, rhi)
    assert_same(dlo, rlo)


def test_submap_insert_one_grid_as_both(ctx):
    """hi and lo the same grid: two rounds, Insert(near) then Insert(all)."""
    p = POSES["tilted"]
    g, r = ctx.grid(0.2), ref.Grid(0.2)
    for returns, origin in _street_local(p):
        ctx.submap_insert_range_data(g, g, p, origin, returns, 20)
        ref.submap_insert(r, r, p, origin, returns, 20)
        assert_same(g, r)


def test_submap_insert_refused_leaves_both_grids(ctx):
    """The high-resolution job alone is valid (16 384 samples at 1 m); the low-resolution job's ray has 32 768 samples at
    0.5 m. The call is refused with DL_ERR_ARG before either grid changes."""
    import dliom
    p = POSES["identity"]
    dhi, dlo, rhi, rlo = submap_pair(ctx, 1.0, 0.5)
    ok = np.array([[3, 1, 0], [5, -2, 1]], f32)
    ctx.submap_insert_range_data(dhi, dlo, p, np.zeros(3, f32), ok, 20)
    ref.submap_insert(rhi, rlo, p, np.zeros(3, f32), ok, 20)
    origin, far = np.array([-12289, 0, 0], f32), np.array([[4095, 0, 0]], f32)
    assert ref.rays(origin, far, 1.0, 2)[3].max() == 16384 and ref.rays(origin, far, 0.5, 2)[3].max() == 32768
    with pytest.raises(dliom.DlError) as e:
        ctx.submap_insert_range_data(dhi, dlo, p, origin, far, 20000)
    assert e.value.status == ref.ERR_ARG
    with pytest.raises(ref.InsertError) as r:
        ref.submap_insert(rhi, rlo, p, origin, far, 20000)
    assert r.value.status == ref.ERR_ARG
    assert_same(dhi, rhi)
    assert_same(dlo, rlo)
    ctx.submap_insert_range_data(dhi, dlo, p, np.zeros(3, f32), ok * 2, 20)   # and the grids take the next Insert
    ref.submap_insert(rhi, rlo, p, np.zeros(3, f32), ok * 2, 20)
    assert_same(dhi, rhi)
    assert_same(dlo, rlo)


# ----------------------------------------------------------------------------------------------- the batched builder
def test_batched_builders_submaps_equal_reference(orc):
    """Three builders through dliom.add_range_data_batch, 15 scans each, num_range_data 3: after every call each inserted
    node's range_data_in_local is replayed through the reference into every submap it went into, at the submap's local pose,
    and every submap's grids (most of them at non-identity poses) must equal the reference's."""
    import dliom
    import synth
    from test_gpu_ltb_batch import Trajectory, feed_imu, make_options
    import imu_synth
    ctx = dliom.Context(0)
    scene = synth.Scene(42)
    trajs = [Trajectory(scene, 2.0 + 0.41 * j) for j in range(3)]
    opts = make_options(orc, num_range_data=3)
    builders = []
    for tr in trajs:
        b = dliom.LocalTrajectoryBuilder(ctx, opts)
        b.set_initial_state(imu_synth.state(tr.t0 - 0.1))
        builders.append(b)
    grids = [dict() for _ in builders]          # submap index -> (reference hi, reference lo)
    io = opts.range_data_inserter
    for step in range(15):
        inputs = []
        for b, tr in zip(builders, trajs):
            t1, imu, xyzt = tr.next()
            feed_imu(b, imu)
            inputs.append((t1, xyzt))
        results = dliom.add_range_data_batch(builders, [t for t, _ in inputs], [x for _, x in inputs])
        for j, (b, r) in enumerate(zip(builders, results)):
            assert r.inserted == 1
            cloud = b.cloud(0)
            origin = np.array(r.origin_in_local, f32)
            for k in range(r.num_insertion_submaps):
                i = r.insertion_submap_index[k]
                pose = b.submap(i)[2]
                if i not in grids[j]:
                    grids[j][i] = (ref.Grid(opts.high_resolution), ref.Grid(opts.low_resolution))
                ref.submap_insert(*grids[j][i], pose, origin, cloud, opts.high_resolution_max_range,
                                  io.hit_probability, io.miss_probability, io.num_free_space_voxels)
            for i, (rhi, rlo) in grids[j].items():
                dhi, dlo = b.submap(i)[:2]
                assert_same(dhi, rhi)
                assert_same(dlo, rlo)
    for j, b in enumerate(builders):
        # a builder may hold a submap that has taken no range data yet: it must be empty
        filled = {i for i in range(b.num_submaps()) if b.submap(i)[3] > 0}
        assert len(filled) >= 5 and set(grids[j]) == filled
        for i in set(range(b.num_submaps())) - filled:
            assert all(len(g.export()[0]) == 0 for g in b.submap(i)[:2])
        assert any(not np.array_equal(b.submap(i)[2], [0, 0, 0, 1, 0, 0, 0]) for i in range(b.num_submaps()))
        b.close()
    ctx.close()
