"""2D probability grids on the device (dl_map_writer_add_probability_grid / _probability_grid) against the reference module
(tests/probability_grid_reference.py): limits (the bits of max), cell counts, the cropped box, every cell value and every
pixel, and the PGM / YAML / PNG bytes. The reference takes each batch as the device writer returns it for that message alone
(one message per call, the same writer settings), so these tests pin the grid stage itself; the map writer's points are
pinned to their own oracle elsewhere, and a writer with grid stages must return the same points, origins and info as one
without."""
import subprocess

import numpy as np
import pytest

import probability_grid_reference as pg
from test_gpu_map_writer import IDENTITY, make_writer, street

pytestmark = pytest.mark.gpu

ROS_FILTER = (1.0, 60.0)                                  # assets_writer_ros_map.lua's min_max_range_filter


@pytest.fixture(scope="module")
def ctx():
    import dliom
    return dliom.Context(0)


def anchored(points_per_msg, origins, stamp0=10_000_000):
    """Messages whose map-frame points are exactly the rows (identity rotation, t = 0, stamp on a node): node k sits at
    origins[k], and a row r of message k lands at r + origins[k] in float."""
    times = np.arange(len(origins), dtype=np.int64) * 1_000_000 + stamp0
    poses = np.array([(o[0], o[1], 0.0, 1.0, 0.0, 0.0, 0.0) for o in origins])
    rows, msgs, first = [], [], 0
    for k, pts in enumerate(points_per_msg):
        pts = np.asarray(pts, np.float32).reshape(-1, 3)
        rows.append(np.concatenate([pts, np.zeros((len(pts), 1), np.float32)], 1))
        msgs.append((int(times[k]), first, len(pts), 0, IDENTITY))
        first += len(pts)
    return {0: (times, poses)}, msgs, np.concatenate(rows + [np.zeros((0, 4), np.float32)])


def run(ctx, trajs, msgs, rows, grids, calls=1, xrays=(), dev=False, **kw):
    """Every pass with the messages split over `calls` calls -> (points, origins, infos, [grid per stage], [xray images])."""
    w = make_writer(ctx, trajs, **kw)
    ids = [w.add_probability_grid(*g) for g in grids]
    xids = [w.add_xray(*x) for x in xrays]
    bounds = np.linspace(0, len(msgs), calls + 1).astype(int)
    if dev:
        import torch
        rows_dev = torch.from_numpy(np.ascontiguousarray(rows)).cuda()
        out_dev = torch.zeros((max(len(rows), 1), 3), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
    while True:
        if dev:
            out = []
            for a, b in zip(bounds[:-1], bounds[1:]):
                n, o, info = w.process_dev(msgs[a:b], rows_dev.data_ptr(), len(rows), out_dev.data_ptr())
                out.append((out_dev[:n].cpu().numpy().copy(), o, info))
        else:
            out = [w.process(msgs[a:b], rows) for a, b in zip(bounds[:-1], bounds[1:])]
        if not w.flush():
            break
    pts = np.concatenate([o[0] for o in out] + [np.zeros((0, 3), np.float32)])
    origins = np.concatenate([o[1] for o in out])
    return pts, origins, [o[2] for o in out], [w.probability_grid(i) for i in ids], [w.xray_image(i) for i in xids]


def batches_of(ctx, trajs, msgs, rows, **kw):
    """The batches the grid stage sees: per message with an origin, (origin, its final-pass points), from a writer without
    stages fed one message per call."""
    w = make_writer(ctx, trajs, **kw)
    while True:
        out = [w.process([m], rows) for m in msgs]
        if not w.flush():
            break
    return [(o[1][0], o[0]) for o in out if not np.isnan(o[1][0][0])]


def reference(batches, resolution, hit, miss, free=True, fast=True):
    return pg.run_batches(resolution, hit, miss, batches, free, fast=fast)


def assert_grid(got, ref):
    info, cells, pixels = got
    want = ref.info()
    assert {k: info[k] for k in want} == want
    assert all(float(info[k]).hex() == float(want[k]).hex() for k in ("resolution", "max_x", "max_y"))
    assert cells.dtype == np.uint16 and cells.tobytes() == np.ascontiguousarray(ref.cropped_cells()).tobytes()
    assert pixels.tobytes() == np.ascontiguousarray(ref.image()).tobytes()


def check(ctx, trajs, msgs, rows, grids, calls=1, fast=True, **kw):
    batches = batches_of(ctx, trajs, msgs, rows, **kw)
    got = run(ctx, trajs, msgs, rows, grids, calls=calls, **kw)[3]
    refs = [reference(batches, *g, fast=fast) for g in grids]
    for g, r in zip(got, refs):
        assert_grid(g, r)
    return batches, got, refs


def ray_fan(rng, n, r_lo, r_hi):
    a = rng.uniform(0, 2 * np.pi, n)
    r = rng.uniform(r_lo, r_hi, n)
    return np.stack([r * np.cos(a), r * np.sin(a), rng.normal(0, 1, n)], 1).astype(np.float32)


def diagonal(sign, n, res=0.05):
    """Points whose superscaled ends at the initial limits are exactly 45 degrees from the origin's (|dx| == |dy|): y on a grid,
    x found by stepping its float until the index matches; sign picks the y direction."""
    ss = pg.Grid(res).limits.superscaled()
    bx, by = ss.cell_index(0.0, 0.0)
    out = []
    for j in range(1, n + 1):
        y = np.float32(j * res)
        want = by + sign * (bx - ss.cell_index(0.0, y)[0])
        x = np.float32(ss.max_x - (want + 0.5) * ss.resolution)
        while ss.cell_index(x, 0.0)[1] != want:
            x = np.nextafter(x, np.float32(np.inf) if ss.cell_index(x, 0.0)[1] > want else np.float32(-np.inf))
        out.append((x, y, np.float32(j)))
    return np.array(out, np.float32)


def shape_edges(shapes, res=0.05):
    """The edges the walk shapes sit on, in the reference's superscaled indices at the initial limits."""
    S = pg.SUBPIXEL
    ss = pg.Grid(res).limits.superscaled()
    b = ss.cell_index(0.0, 0.0)
    ends = {name: [ss.cell_index(p[0], p[1]) for p in pts] for name, pts in shapes.items()}
    assert all(e[0] // S == b[0] // S for e in ends["column"])                                   # the vertical special case
    assert all(e[1] // S == b[1] // S and e[0] // S != b[0] // S for e in ends["row"])           # dy = 0 in pixels
    assert (b[0] % S) == (b[1] % S)
    signs = set()
    for name in ("corner_up", "corner_down"):                                                    # through pixel corners
        assert all(abs(e[0] - b[0]) == abs(e[1] - b[1]) for e in ends[name])
        signs |= {(np.sign(e[0] - b[0]), np.sign(e[1] - b[1])) for e in ends[name]}
    assert len(signs) == 2                                                                       # both y directions
    assert ends["near"][0] == b and ends["near"][1][0] // S == b[0] // S                          # one subpixel, one pixel
    assert ends["near"][1][1] // S == b[1] // S
    octants = {(np.sign(e[0] - b[0]), np.sign(e[1] - b[1]), abs(e[0] - b[0]) > abs(e[1] - b[1])) for e in ends["octants"]}
    assert len(octants) == 8
    hits = {(e[0] // S, e[1] // S) for e in ends["collinear"]}
    walked = set()
    pg.cast_ray(b, ends["collinear"][-1], lambda x, y: walked.add((x, y)))
    assert len(hits & walked) >= 3                                                               # hits crossed by a walk


def walk_shapes():
    k = np.arange(1, 40, dtype=np.float32)[:, None]
    return {   # all but the octants stay inside the first 100 x 100 cells: their ends are read at the initial limits
        # superscaled x comes from the y coordinate: y = 0 keeps the origin's pixel column, x = -0.01 its pixel row
        "column": np.concatenate([k * np.float32(0.05) * (-1) ** k, np.zeros_like(k), k], 1),
        "row": np.concatenate([np.full_like(k, -0.01), k * np.float32(0.05) * (-1) ** k, k], 1),
        "corner_up": diagonal(1, 39),
        "corner_down": diagonal(-1, 39),
        "near": np.array([[-1e-6, -1e-6, 0], [-0.01, -0.02, 0], [-0.03, -0.04, 0], [0, 0, 5]], np.float32),
        "collinear": np.array([[x, 0.3 * x, 0] for x in (0.4, 0.8, 1.2, 1.6, 2.0)], np.float32),
        "octants": ray_fan(np.random.default_rng(1), 400, 0.1, 3.0),
    }


def test_walk_shapes_sit_on_their_edges(ctx):
    """Octants, axis-aligned walks (one pixel column and dy = 0), 45-degree walks through pixel corners in both y directions,
    ends in the origin's pixel and subpixel, and hit cells crossed by other walks of the same batch."""
    shapes = walk_shapes()
    shape_edges(shapes)
    trajs, msgs, rows = anchored(list(shapes.values()), [(0.0, 0.0)] * len(shapes))
    _, _, refs = check(ctx, trajs, msgs, rows, [(0.05, 0.55, 0.49)], fast=False)
    # every hit cell holds the hit table's value (a hit wins over the misses of its batch)
    hit_value = int(pg.correspondence_cost_table(0.55)[0]) - pg.UPDATE_MARKER
    g = refs[0]
    assert g.cells[(hit_value == g.cells)].size >= 4


def test_rounding_boundaries_one_ulp_either_side(ctx):
    """Float points whose superscaled quotient lies just below and just above a .5 rounding boundary."""
    res = 0.05
    ss = pg.Grid(res).limits.superscaled()
    pairs = []
    for k in range(10_000, 90_000, 1_999):
        y = np.float32(ss.max_y - (k + 1) * ss.resolution)          # near (max - y) / res - 0.5 = k + 0.5
        for _ in range(4):
            y = np.nextafter(y, np.float32(-np.inf))
        for _ in range(8):
            nxt = np.nextafter(y, np.float32(np.inf))
            if ss.cell_index(0.0, y)[0] != ss.cell_index(0.0, nxt)[0]:
                pairs.append((y, nxt))
                break
            y = nxt
    assert len(pairs) > 30
    pts = [[0.3, float(a), 0] for a, _ in pairs] + [[0.3, float(b), 0] for _, b in pairs]
    pts += [[float(a), -0.4, 0] for a, _ in pairs] + [[float(b), -0.4, 0] for _, b in pairs]
    trajs, msgs, rows = anchored([pts], [(0.0, 0.0)])
    check(ctx, trajs, msgs, rows, [(res, 0.55, 0.49)], fast=False)


def test_one_cell_crossed_by_many_walks_and_many_batches(ctx):
    rng = np.random.default_rng(2)
    one = [ray_fan(rng, 100_000, 0.5, 4.0)]
    trajs, msgs, rows = anchored(one, [(0.013, -0.021)])
    check(ctx, trajs, msgs, rows, [(0.05, 0.55, 0.49)])
    many = [ray_fan(rng, 8, 0.5, 2.0) for _ in range(1000)]
    trajs, msgs, rows = anchored(many, [(0.013, -0.021)] * 1000)
    _, got, refs = check(ctx, trajs, msgs, rows, [(0.05, 0.55, 0.49), (0.1, 0.7, 0.3, False)])
    centre = refs[0].limits.cell_index(0.013, -0.021)
    assert refs[0].cells[centre[1], centre[0]] == 32767                   # 1000 misses drive the origin cell's cost to the top


def test_growth_none_once_many_each_direction_and_between_batches(ctx):
    rng = np.random.default_rng(4)
    small = ray_fan(rng, 50, 0.1, 2.0)                                     # inside the first 100 x 100 cells at 5 cm
    cases = [[small], [small + np.float32([2.0, 0, 0])], [small * np.float32(30.0)]]
    for d in ([6.0, 0], [-6.0, 0], [0, 6.0], [0, -6.0]):
        cases.append([small + np.float32(d + [0])])
    sizes = []
    for pts in cases:
        trajs, msgs, rows = anchored(pts, [(0.0, 0.0)])
        _, got, refs = check(ctx, trajs, msgs, rows, [(0.05, 0.55, 0.49)])
        sizes.append(got[0][0]["num_x_cells"])
    assert sizes[:2] == [100, 200] and sizes[2] >= 1600 and min(sizes[3:]) >= 400
    # batches of one call at different limits, and the same stream over several calls
    walk = [ray_fan(rng, 200, 0.5, 3.0) for _ in range(12)]
    origins = [(3.0 * k * (-1) ** k, 2.5 * k, 0.0) for k in range(12)]
    trajs, msgs, rows = anchored(walk, origins)
    sizes = {r.limits.num_x for r in [reference(batches_of(ctx, trajs, msgs[:k], rows), 0.05, 0.55, 0.49)
                                     for k in (1, 4, 8, 12)]}
    assert len(sizes) >= 3
    for calls in (1, 3, 12):
        check(ctx, trajs, msgs, rows, [(0.05, 0.55, 0.49)], calls=calls)


def test_growth_by_the_origin_of_an_emptied_batch(ctx):
    """The range filter empties the second message (its points lie within 1 m of its origin 20 m away): the batch still grows
    the grid to take in its origin."""
    rng = np.random.default_rng(6)
    close = ray_fan(rng, 30, 0.1, 0.5)
    close[:, 2] = 0.0                                                     # every point within 0.5 m of its origin
    trajs, msgs, rows = anchored([ray_fan(rng, 100, 1.5, 2.0), close], [(0.0, 0.0), (20.0, -15.0)])
    batches, got, refs = check(ctx, trajs, msgs, rows, [(0.05, 0.55, 0.49)], range_filter=(1.0, 60.0))
    assert len(batches) == 2 and len(batches[1][1]) == 0 and got[0][0]["num_x_cells"] > 400


def test_moving_object_removal_and_xray_stages_alongside(ctx):
    """Two grid stages (0.05 and 0.1 m) next to the X-ray backpack stages on the street with the transient box; the final pass
    only. Points, origins, info and the X-ray images equal those of writers without the grid stages."""
    from test_gpu_xray import XY, XZ, YZ
    trajs, msgs, rows = street(num_scans=10, transient_scans=4)
    kw = dict(range_filter=(1.0, 40.0), outlier_voxel_size=0.2)
    xrays = [(0.05, YZ), (0.05, XY), (0.05, XZ)]
    grids = [(0.05, 0.55, 0.49), (0.1, 0.6, 0.45)]
    pts, origins, infos, got, images = run(ctx, trajs, msgs, rows, grids, xrays=xrays, **kw)
    base = run(ctx, trajs, msgs, rows, [], xrays=xrays, **kw)
    assert pts.tobytes() == base[0].tobytes() and origins.tobytes() == base[1].tobytes() and infos == base[2]
    assert all(a.tobytes() == b.tobytes() for a, b in zip(images, base[4]))
    assert infos[0]["dropped_moving"] > 0
    batches = batches_of(ctx, trajs, msgs, rows, **kw)
    for g, spec in zip(got, grids):
        assert_grid(g, reference(batches, *spec))


def test_calls_and_device_buffers_are_byte_identical(ctx):
    trajs, msgs, rows = street(num_scans=8, transient_scans=0)
    grids = [(0.05, 0.55, 0.49)]
    one = run(ctx, trajs, msgs, rows, grids, range_filter=ROS_FILTER)
    for calls, dev in ((3, False), (8, False), (1, True), (4, True)):
        other = run(ctx, trajs, msgs, rows, grids, calls=calls, dev=dev, range_filter=ROS_FILTER)
        assert other[0].tobytes() == one[0].tobytes()
        assert other[3][0][0] == one[3][0][0]
        assert other[3][0][1].tobytes() == one[3][0][1].tobytes() and other[3][0][2].tobytes() == one[3][0][2].tobytes()


@pytest.mark.parametrize("beams,scans", [(16, 12), (64, 3)])
def test_ros_map_pipeline_on_street_drives(ctx, tmp_path, beams, scans):
    """assets_writer_ros_map.lua: min_max_range_filter 1-60 m, then write_ros_map at 0.05 m (hit 0.55, miss 0.49): every cell,
    and the PGM / YAML / PNG bytes."""
    import dliom
    trajs, msgs, rows = street(num_scans=scans, transient_scans=0, beams=beams)
    batches, got, refs = check(ctx, trajs, msgs, rows, [(0.05, 0.55, 0.49)], range_filter=ROS_FILTER)
    info, cells, pixels = got[0]
    assert (cells != 0).sum() > 20_000 and (pixels < 128).any() and (pixels > 128).any()   # occupied darker, free lighter
    stem = str(tmp_path / "map")
    dliom.write_ros_map(stem, info, pixels)
    pgm, yaml = pg.ros_map(refs[0].info(), refs[0].image(), stem + ".pgm")
    assert open(stem + ".pgm", "rb").read() == pgm and open(stem + ".yaml", "rb").read() == yaml
    dliom.write_probability_grid_png(str(tmp_path / "grid.png"), pixels)
    assert open(tmp_path / "grid.png", "rb").read() == dliom.png_bytes(dliom.grey_argb(refs[0].image()))


def test_insert_free_space_false_and_empty_grids(ctx):
    rng = np.random.default_rng(8)
    trajs, msgs, rows = anchored([ray_fan(rng, 300, 0.5, 3.0)], [(0.0, 0.0)])
    _, got, refs = check(ctx, trajs, msgs, rows, [(0.05, 0.55, 0.49, False)])
    assert set(np.unique(got[0][1]).tolist()) <= {0, int(pg.correspondence_cost_table(0.55)[0]) - pg.UPDATE_MARKER}
    # no batch at all, and a batch without points: offset 0, 1 x 1, one unknown cell, grey 128
    for pts, kw in (([], {}), ([np.zeros((3, 3), np.float32)], dict(range_filter=(1.0, 60.0)))):
        t, m, r = anchored(pts, [(0.0, 0.0)] * max(len(pts), 1))
        info, cells, pixels = run(ctx, t, m, r, [(0.05, 0.55, 0.49)], **kw)[3][0]
        assert (info["offset_x"], info["offset_y"], info["width"], info["height"]) == (0, 0, 1, 1)
        assert cells.tolist() == [[0]] and pixels.tolist() == [[128]]


def test_rejections_leave_the_writer_unchanged(ctx):
    import ctypes as C
    import dliom
    rng = np.random.default_rng(9)
    good = [ray_fan(rng, 200, 0.5, 3.0) for _ in range(3)]
    far = [np.float32([[1.0, 0, 0], [1e6, 0.0, 0]]), np.float32([[1.0, 0, 0], [np.inf, 0.0, 0]]),
           np.float32([[1.0, 0, 0], [0.0, np.nan, 0]])]
    trajs, msgs, rows = anchored(good + far, [(0.0, 0.0)] * 6)
    w = make_writer(ctx, trajs)
    for bad in ((0.0, 0.55, 0.49), (-0.05, 0.55, 0.49), (float("nan"), 0.55, 0.49), (float("inf"), 0.55, 0.49),
                (0.05, 0.5, 0.49), (0.05, 0.55, 0.5), (0.05, float("nan"), 0.49), (0.05, 0.55, float("nan"))):
        with pytest.raises(dliom.DlError) as e:
            w.add_probability_grid(*bad)
        assert e.value.status == -2
    s = w.add_probability_grid(0.05, 0.55, 0.49)
    with pytest.raises(dliom.DlError):
        w.probability_grid(s)                                    # before the final flush
    # growth past 100 * 2^14 cells and non-finite points, each refused with nothing changed
    for k in (3, 4, 5):
        with pytest.raises(dliom.DlError) as e:
            w.process(msgs[:2] + [msgs[k]], rows)
        assert e.value.status == -2
    w.process(msgs[:3], rows)
    with pytest.raises(dliom.DlError):
        w.add_probability_grid(0.05, 0.55, 0.49)                 # after processing began
    assert w.flush() is False
    with pytest.raises(dliom.DlError):
        w.probability_grid(1)                                    # unknown stage
    info = dliom.MapWriterGridInfo()
    small = np.zeros(1, np.uint16)
    assert ctx.L.dl_map_writer_probability_grid(w.h, 0, C.byref(info), 1, small.ctypes.data, None) == -2
    batches = [(np.zeros(3, np.float32), g) for g in good]
    assert_grid(w.probability_grid(s), reference(batches, 0.05, 0.55, 0.49))
    # the stage cap counts grid stages with the X-ray and colour stages
    c = make_writer(ctx, trajs)
    for k in range(8):
        c.add_probability_grid(0.1 * (k + 1), 0.55, 0.49)
        c.add_color(k, (k, k, k))
    with pytest.raises(dliom.DlError):
        c.add_probability_grid(0.05, 0.55, 0.49)
    with pytest.raises(dliom.DlError):
        c.add_xray(1.0, IDENTITY)


def test_cpp_example_writes_the_same_files(ctx, tmp_path):
    """build/example_ros_map (io::MapWriter, RosMapWritingPointsProcessor, ProbabilityGridPointsProcessor) writes map.pgm,
    map.yaml and probability_grid.png, byte for byte those of the Python writers over dliom.MapWriter on the same input."""
    import dliom
    import __graft_entry__
    from test_map_writer_oracle import write_map_input
    trajs, msgs, rows = street(num_scans=8, transient_scans=3)
    kw = dict(range_filter=ROS_FILTER, outlier_voxel_size=0.2)
    path = str(tmp_path / "input.bin")
    write_map_input(path, trajs, msgs, rows, range_filter=kw["range_filter"], voxel_size=kw["outlier_voxel_size"])
    out = tmp_path / "cpp"
    out.mkdir()
    r = subprocess.run([__graft_entry__.ROS_MAP_EXAMPLE, path, str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    pts, _, _, grids, _ = run(ctx, trajs, msgs, rows, [(0.05, 0.55, 0.49)] * 2, **kw)
    info, _, pixels = grids[0]
    assert r.stdout.split("\n")[:2] == [f"points {len(pts)}", f"grid {info['width']} {info['height']}"]
    stem = str(out / "map")
    pgm, yaml = dliom.ros_map_bytes(info, pixels, stem + ".pgm")
    assert (out / "map.pgm").read_bytes() == pgm and (out / "map.yaml").read_bytes() == yaml
    assert (out / "probability_grid.png").read_bytes() == dliom.png_bytes(dliom.grey_argb(grids[1][2]))
