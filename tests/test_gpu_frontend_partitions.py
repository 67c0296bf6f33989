"""The fused front half merges each voxel filter's tile winners by hash partition (dl_frontend.cu, kernels A2 and B2): every
tile writes its winners to the scan's partitions, and one CTA per (scan, partition) keeps the lowest index per voxel in shared
memory, or, when the partition holds more than one tile's worth of entries, in a global table of its own. Every case compares
the survivors and their order with the oracle's ingest_scan, bit for bit: the largest partitions (every row its own voxel), one
voxel over many tiles, scan sizes around a tile and at the batch's capacity, an empty scan inside a batch, the three row
formats, and a scan built so that one partition of each filter overflows its shared table."""
import numpy as np
import pytest

from helpers import workload

pytestmark = pytest.mark.gpu

TILE = 2048        # rows per tile; also the most entries a partition merges in shared memory
MAX_PARTS = 256    # most partitions per scan


def hash_cell(c):
    """dl_frontend.cu hash_cell over an (n, 3) int array, in wrapping 32-bit arithmetic."""
    c = c.astype(np.int64).astype(np.uint32)
    with np.errstate(over="ignore"):
        h = (c[:, 0] * np.uint32(73856093)) ^ (c[:, 1] * np.uint32(19349663)) ^ (c[:, 2] * np.uint32(83492791))
        h ^= h >> np.uint32(15)
        h *= np.uint32(0x2C1B3C6D)
        h ^= h >> np.uint32(12)
    return h


def num_parts(n):
    return min(2 * ((n + TILE - 1) // TILE), MAX_PARTS)


def first_part(cells, parts):
    """Partition of a first-filter cell: the hash's low 20 bits (the tile table takes the top 12)."""
    h = (hash_cell(cells).astype(np.uint64) << np.uint64(12)) & np.uint64(0xFFFFFFFF)
    return ((h * np.uint64(parts)) >> np.uint64(32)).astype(np.int64)


def second_part(cells, parts):
    """Partition of a second-filter return's cell: hash bits 12..31 (the tile table takes the low 12)."""
    h = hash_cell(cells).astype(np.uint64) & np.uint64(0xFFFFF000)
    return ((h * np.uint64(parts)) >> np.uint64(32)).astype(np.int64)


@pytest.fixture(scope="module")
def ctx():
    import dliom
    c = dliom.Context(0)
    yield c
    c.close()


def assert_ingest_equal(ctx, orc, w, rows, prev, cur):
    import dliom
    fo = dliom.FrontendOptions.from_oracle(w["opts"])
    want = orc.ingest_scan(w["opts"], rows, w["origin"], prev, cur)
    got = ctx.ingest_scan(fo, rows, w["origin"], prev, cur)
    assert np.array_equal(got["first_keep"], want["first_keep"])
    for k in ("returns_local", "returns_tracking", "misses_tracking", "current_pose"):
        assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), k
    return want


def still_rows(w, xyz):
    """32-byte rows at the given points, every time 0 (no deskew), all from origin 0."""
    rows = np.zeros(len(xyz), w["scans"][0].dtype)
    rows["x"], rows["y"], rows["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    return rows


def test_every_row_its_own_voxel_in_random_order(ctx, orc):
    """20 tiles of distinct voxels in both filters: every row is a tile winner and a survivor, the largest partitions."""
    w = workload()
    s = np.float32(w["opts"].voxel_filter_size)
    g = np.arange(-110, 110, dtype=np.float32)
    x, y = np.meshgrid(g, g, indexing="ij")
    xyz = np.stack([x.ravel(), y.ravel(), np.full(x.size, 20.0, np.float32)], 1)[: 20 * TILE] * s
    xyz = xyz[np.random.default_rng(11).permutation(len(xyz))]
    ident = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
    want = assert_ingest_equal(ctx, orc, w, still_rows(w, xyz), ident, ident)
    assert len(want["first_keep"]) == 20 * TILE


def test_one_voxel_over_many_tiles(ctx, orc):
    """Every row of 20 tiles in one voxel: each tile has one winner, and all meet in one partition."""
    w = workload()
    base = w["scans"][0]
    rows = np.resize(base, 20 * TILE + 5).copy()
    for k in "xyz":
        rows[k] = base[k][100]
    want = assert_ingest_equal(ctx, orc, w, rows, w["prev"][0], w["cur"][0])
    assert len(want["first_keep"]) == 1


@pytest.mark.parametrize("size", [1, TILE - 1, TILE, TILE + 1, None])
def test_scan_sizes(ctx, orc, size):
    """None: a whole 64-beam sweep (the scan is the call's capacity)."""
    w = workload(beams=64, num_map_scans=4, num_scans=1)
    rows = w["scans"][0]
    assert_ingest_equal(ctx, orc, w, (rows if size is None else rows[:size]).copy(), w["prev"][0], w["cur"][0])


def test_batch_sizes_formats_and_empty_scan(ctx, orc):
    """One batch at the capacity of its longest scan, with scans of 1, 2047, 2048 and 2049 rows and an empty one, in the 12-,
    16- and 32-byte row formats: the oracle's survivor counts, and the same result in every format."""
    import dliom
    w = workload(beams=64, num_map_scans=4, num_scans=4)
    hi, lo = dliom.Grid.from_oracle(ctx, w["hi"]), dliom.Grid.from_oracle(ctx, w["lo"])
    full = w["scans"][0]
    scans = [full.copy(), full[:1].copy(), full[:TILE - 1].copy(), full[:0].copy(), full[:TILE].copy(),
             full[:TILE + 1].copy()]
    scans = [s[np.random.default_rng(k).permutation(len(s))].copy() for k, s in enumerate(scans)]
    prev, cur = w["prev"][[0] * len(scans)], w["cur"][[0] * len(scans)]
    r4 = [np.ascontiguousarray(np.stack([s[k] for k in "xyzt"], 1)) for s in scans]
    r3 = [np.ascontiguousarray(r[:, :3]) for r in r4]
    fo8 = dliom.FrontendOptions.from_oracle(w["opts"])
    fo4 = dliom.FrontendOptions.from_oracle(w["opts"])
    fo4.range_row_floats = 4
    fo3 = dliom.FrontendOptions.from_oracle(w["opts"])
    dliom.TimeRuns([s["t"] for s in scans]).attach(fo3)
    args = (w["origin"], prev, cur, w["submap_pose"], hi, lo)
    got = [ctx.frontend_match_batch(fo8, scans, *args), ctx.frontend_match_batch(fo4, r4, *args),
           ctx.frontend_match_batch(fo3, r3, *args)]
    for s, rows in enumerate(scans):
        if len(rows) == 0:
            assert all((r[s].num_first_filter, r[s].num_returns, r[s].num_misses) == (0, 0, 0) for r in got)
            continue
        ing = orc.ingest_scan(w["opts"], rows, w["origin"], prev[s], cur[s])
        want = (len(ing["first_keep"]), len(ing["returns_tracking"]), len(ing["misses_tracking"]))
        for r in got:
            assert (r[s].num_first_filter, r[s].num_returns, r[s].num_misses) == want, s
            assert r[s].ok == got[0][s].ok
            assert list(r[s].pose_estimate_local) == list(got[0][s].pose_estimate_local), s


def test_partition_overflows_its_shared_table(ctx, orc):
    """2 600 distinct voxels whose hashes fall in partition 0 of both filters (found here with the kernels' hash), then 1 000 of
    them again (they lose in the first filter's merge) and 500 of them shifted by 0.4 voxel along x (a first-filter voxel of
    their own, but they lose in the second filter's merge). Partition 0 holds more than the TILE entries a shared table merges
    in both filters, so both merges take their global table."""
    w = workload()
    s = np.float32(w["opts"].voxel_filter_size)
    n = 2600 + 1000 + 500
    parts = num_parts(n)
    g = np.arange(10, 60)
    c2 = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)   # second-filter cells; the first filter's are 2 c2
    pick = c2[(first_part(2 * c2, parts) == 0) & (second_part(c2, parts) == 0)]
    assert len(pick) >= 2600
    pick = pick[np.random.default_rng(5).permutation(len(pick))[:2600]].astype(np.float32)
    shifted = pick[:500] + np.array([0.4, 0, 0], np.float32)
    xyz = np.concatenate([pick, pick[:1000], shifted]) * s
    assert len(xyz) == n and np.all(np.linalg.norm(xyz, axis=1) <= w["opts"].max_range)
    first_cells = np.rint(xyz / np.float32(0.5 * s)).astype(np.int64)
    second_cells = np.rint(xyz / s).astype(np.int64)
    assert np.array_equal(first_cells[:3600], 2 * np.concatenate([pick, pick[:1000]]).astype(np.int64))
    assert np.array_equal(second_cells[3600:], pick[:500].astype(np.int64))
    # entries per partition: every row of the first tile; later tiles add their tile winners (of the first filter's survivors)
    assert np.bincount(first_part(first_cells, parts), minlength=parts)[0] >= 3600 > TILE
    keep = np.r_[0:2600, 3600:n]
    assert np.bincount(second_part(second_cells[keep], parts), minlength=parts)[0] == 3100 > TILE
    ident = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
    want = assert_ingest_equal(ctx, orc, w, still_rows(w, xyz), ident, ident)
    assert np.array_equal(want["first_keep"], keep)
    assert len(want["returns_tracking"]) == 2600
