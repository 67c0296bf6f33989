"""The fused front half de-duplicates both voxel filters per tile of 2048 consecutive rows before it touches the scan-wide tables
(dl_frontend.cu). Rows in firing order make that cheap; correctness must not depend on it. Every case here compares the fused
front end against the oracle chain on inputs that defeat the tiling: rows in random order, voxels split between the first and
the last tile, scans one row around a tile boundary, a scan that is one voxel, a scan of distinct voxels (a full tile table),
an empty scan, the key-range flag raised inside a tile, and the 12-, 16- and 32-byte row formats with and without deskew."""
import numpy as np
import pytest

from helpers import workload

pytestmark = pytest.mark.gpu

TILE = 2048


@pytest.fixture(scope="module")
def ctx():
    import dliom
    c = dliom.Context(0)
    yield c
    c.close()


def assert_ingest_equal(ctx, orc, w, rows, s=0):
    """dl_ingest_scan runs the fused kernels (and checks their counts against the stage-wise ones); the tracking-frame clouds
    and the current pose come from the fused path."""
    import dliom
    fo = dliom.FrontendOptions.from_oracle(w["opts"])
    want = orc.ingest_scan(w["opts"], rows, w["origin"], w["prev"][s], w["cur"][s])
    got = ctx.ingest_scan(fo, rows, w["origin"], w["prev"][s], w["cur"][s])
    assert np.array_equal(got["first_keep"], want["first_keep"])
    for k in ("returns_local", "returns_tracking", "misses_tracking", "current_pose"):
        assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), k
    return want


def test_full_size_scan_in_random_order(ctx, orc):
    w = workload(beams=64, num_map_scans=6, num_scans=3)
    rows = w["scans"][0]
    shuffled = rows[np.random.default_rng(3).permutation(len(rows))].copy()
    want = assert_ingest_equal(ctx, orc, w, shuffled)
    assert len(want["first_keep"]) > 20000


def test_voxels_split_between_first_and_last_tile(ctx, orc):
    w = workload()
    rows = w["scans"][1].copy()
    n = len(rows)
    assert n > 8 * TILE
    for k in range(8):                  # rows of the first tile repeated at the end of the scan, and the other way round
        rows[n - 1 - k] = rows[3 * k]
        rows[TILE - 1 - k] = rows[n - 20 - 3 * k]
    assert_ingest_equal(ctx, orc, w, rows, s=1)


@pytest.mark.parametrize("size", [TILE - 1, TILE, TILE + 1, 2 * TILE + 1, 1])
def test_scan_sizes_around_a_tile(ctx, orc, size):
    w = workload()
    assert_ingest_equal(ctx, orc, w, w["scans"][2][:size].copy(), s=2)


def test_one_voxel_and_distinct_voxels(ctx, orc):
    w = workload()
    base = w["scans"][0]
    one = base[:3 * TILE + 7].copy()
    for k in "xyz":
        one[k] = base[k][100]            # every row in the same first-filter voxel; the times still spread the deskew
    assert_ingest_equal(ctx, orc, w, one)
    g = np.arange(-32, 32, dtype=np.float32) * 0.5 + 0.25
    x, y = np.meshgrid(g, g, indexing="ij")
    distinct = np.resize(base, x.size).copy()  # 4 096 rows, every one its own voxel in both filters (two full tiles)
    distinct["x"], distinct["y"], distinct["z"] = x.ravel(), y.ravel(), np.float32(1.25)
    want = assert_ingest_equal(ctx, orc, w, distinct)
    assert len(want["first_keep"]) == x.size


def rows_formats(scans):
    import dliom
    r4 = [np.ascontiguousarray(np.stack([s[k] for k in "xyzt"], 1)) for s in scans]
    return r4, [np.ascontiguousarray(r[:, :3]) for r in r4], dliom.TimeRuns([s["t"] for s in scans])


@pytest.mark.parametrize("deskew", [True, False])
def test_row_formats_and_empty_scan(ctx, orc, deskew):
    """12-, 16- and 32-byte rows give the oracle's counts and the same pose, bit for bit, with an empty scan in the batch."""
    import dliom
    w = workload()
    hi, lo = dliom.Grid.from_oracle(ctx, w["hi"]), dliom.Grid.from_oracle(ctx, w["lo"])
    rng = np.random.default_rng(7)
    scans = [w["scans"][0][rng.permutation(len(w["scans"][0]))].copy(), w["scans"][1][:TILE + 1].copy(),
             w["scans"][2][:0].copy(), w["scans"][3].copy()]
    if not deskew:
        for s in scans:
            s["t"] = 0.0                 # LTB:430-433: |t_0| < 1e-3 -> no deskew
    r4, r3, runs = rows_formats(scans)
    args = (w["origin"], w["prev"], w["cur"], w["submap_pose"], hi, lo)
    fo8 = dliom.FrontendOptions.from_oracle(w["opts"])
    fo4 = dliom.FrontendOptions.from_oracle(w["opts"])
    fo4.range_row_floats = 4
    fo3 = dliom.FrontendOptions.from_oracle(w["opts"])
    runs.attach(fo3)
    got = [ctx.frontend_match_batch(fo8, scans, *args), ctx.frontend_match_batch(fo4, r4, *args),
           ctx.frontend_match_batch(fo3, r3, *args)]
    for s, rows in enumerate(scans):
        if len(rows) == 0:
            assert all((r[s].num_first_filter, r[s].num_returns, r[s].num_misses) == (0, 0, 0) for r in got)
            continue
        ing = orc.ingest_scan(w["opts"], rows, w["origin"], w["prev"][s], w["cur"][s])
        want = (len(ing["first_keep"]), len(ing["returns_tracking"]), len(ing["misses_tracking"]))
        for r in got:
            assert (r[s].num_first_filter, r[s].num_returns, r[s].num_misses) == want, s
            assert r[s].ok == got[0][s].ok
            assert list(r[s].pose_estimate_local) == list(got[0][s].pose_estimate_local), s


def test_key_range_flag_inside_a_tile(ctx, orc):
    """One point beyond the key span of a 0.4 mm second filter, in the middle of a tile, invalidates that scan only."""
    import dliom
    w = workload()
    hi, lo = dliom.Grid.from_oracle(ctx, w["hi"]), dliom.Grid.from_oracle(ctx, w["lo"])
    fo = dliom.FrontendOptions.from_oracle(w["opts"])
    fo.range_row_floats = 4
    fo.voxel_filter_size = 4e-4
    full = np.ascontiguousarray(np.stack([w["scans"][0][k] for k in "xyzt"], 1))
    far = np.linalg.norm(full[:, :3], axis=1) > 20.0
    near = np.ascontiguousarray(full[~far])
    near = np.ascontiguousarray(near[np.linalg.norm(near[:, :3], axis=1) < 5.0])
    near[-1, 3] = 0.0
    assert len(near) > 500
    flagged = near.copy()
    flagged[len(near) // 2, :3] = full[far][0, :3]
    res = ctx.frontend_match_batch(fo, [near, flagged, near], w["origin"], w["prev"][[0, 0, 0]], w["cur"][[0, 0, 0]],
                                   w["submap_pose"], hi, lo)
    assert (res[0].ok, res[1].ok, res[2].ok) == (1, -1, 1)
