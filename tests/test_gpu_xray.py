"""X-ray images and point colours on the device (dl_map_writer_add_xray / _add_color / _xray_image) against the CPU oracle
(tests/xray_oracle.py), every image word bit for bit: the reference's backpack pipeline on the street scene with range filter and
moving-object removal, non-dyadic colours interleaved within columns, the stream split over many calls, the device-buffer entry
point, each rejection with the writer unchanged, map-writer outputs with and without stages, and the C++ example's PNG files."""
import math
import subprocess

import numpy as np
import pytest

import map_writer_oracle as mo
import xray_oracle as xo
from test_gpu_map_writer import IDENTITY, make_writer, oracle_trajs, street

pytestmark = pytest.mark.gpu


def rotation(roll, pitch, yaw):
    import dliom
    return (0.0, 0.0, 0.0) + tuple(dliom.roll_pitch_yaw(roll, pitch, yaw))


XY, XZ, YZ = rotation(0.0, -math.pi / 2.0, 0.0), rotation(0.0, 0.0, -math.pi / 2), rotation(0.0, 0.0, math.pi)
VOXEL = 5e-2
# assets_writer_backpack_3d.lua after its range filter; frame 0 = horizontal_vlp16_link, frame 1 = vertical_vlp16_link
BACKPACK = [("xray", VOXEL, YZ), ("xray", VOXEL, XY), ("xray", VOXEL, XZ), ("color", 0, (255, 0, 0)), ("color", 1, (0, 255, 0)),
            ("xray", VOXEL, YZ), ("xray", VOXEL, XY), ("xray", VOXEL, XZ)]


@pytest.fixture(scope="module")
def ctx():
    import dliom
    return dliom.Context(0)


def add_stages(w, stages):
    return [w.add_xray(s[1], s[2]) if s[0] == "xray" else w.add_color(s[1], s[2]) for s in stages]


def run(ctx, trajs, msgs, rows, stages, calls=1, **kw):
    """Every pass with the messages split over `calls` calls -> (final points, origins, infos, images)."""
    w = make_writer(ctx, trajs, **kw)
    ids = [i for i in add_stages(w, stages) if i is not None]
    bounds = np.linspace(0, len(msgs), calls + 1).astype(int)
    while True:
        out = [w.process(msgs[a:b], rows) for a, b in zip(bounds[:-1], bounds[1:])]
        if not w.flush():
            break
    pts = np.concatenate([o[0] for o in out])
    return pts, np.concatenate([o[1] for o in out]), [o[2] for o in out], [w.xray_image(i) for i in ids]


def with_frames(msgs, frames):
    return [m + (frames[k % len(frames)],) for k, m in enumerate(msgs)]


def oracle_images(trajs, msgs, rows, stages, range_filter=None, voxel_size=0.0):
    res, frames = xo.final_pass(oracle_trajs(trajs), msgs, rows, range_filter, voxel_size)
    return res, xo.xray_images(res["points"], frames, stages)


def assert_images(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.shape == w.shape and g.tobytes() == w.tobytes()


def test_backpack_pipeline_matches_the_oracle_on_the_street(ctx):
    trajs, msgs, rows = street()
    msgs = with_frames(msgs, (0, 1))
    kw = dict(range_filter=(1.0, 40.0), outlier_voxel_size=0.2)
    pts, origins, infos, images = run(ctx, trajs, msgs, rows, BACKPACK, **kw)
    res, want = oracle_images(trajs, msgs, rows, BACKPACK, (1.0, 40.0), 0.2)
    assert pts.tobytes() == res["points"].tobytes() and res["dropped_moving"] > 0
    assert_images(images, want)
    gray, color = images[:3], images[3:]
    for g, c in zip(gray, color):
        assert g.shape == c.shape and g.shape[0] > 20 and g.shape[1] > 20
        assert (g != xo.WHITE).sum() > 1000
        r, gr = (c >> 16) & 0xFF, (c >> 8) & 0xFF
        assert (r > gr).any() and (gr > r).any()        # both LiDARs' colours show
    # the same writer without stages: the same points, origins and info
    base = make_writer(ctx, trajs, **kw)
    while True:
        b = base.process(msgs, rows)
        if not base.flush():
            break
    assert b[0].tobytes() == pts.tobytes() and b[1].tobytes() == origins.tobytes() and b[2] == infos[0]


def test_interleaved_non_dyadic_colours_and_many_calls(ctx):
    trajs, msgs, rows = street(num_scans=12, transient_scans=0)
    msgs = with_frames(msgs, (2, 5, 2, 9))
    stages = [("color", 2, (128, 77, 3)), ("xray", 0.1, XY), ("color", 5, (3.7, 200, 77)), ("color", 2, (1, 254, 128)),
              ("xray", VOXEL, XZ), ("xray", 0.03, (0.5, -0.25, 1.0) + XY[3:])]
    res, want = oracle_images(trajs, msgs, rows, stages, (1.0, 60.0))
    for calls in (1, 5, 12):
        _, _, _, images = run(ctx, trajs, msgs, rows, stages, calls=calls, range_filter=(1.0, 60.0))
        assert_images(images, want)


def test_column_sum_order_across_calls(ctx):
    """774 one-point messages into one column of two voxels, frames alternating red 255 / 128: summed out of stream order the
    mean lands one byte higher (tests/test_xray_oracle.py)."""
    trajs = {0: (np.array([0], np.int64), np.array([IDENTITY]))}
    n = 774
    rows = np.zeros((n, 4), np.float32)
    rows[1::2, 0] = 1.0
    msgs = [(0, k, 1, 0, IDENTITY, k % 2) for k in range(n)]
    stages = [("color", 0, (255, 0, 0)), ("color", 1, (128, 0, 0)), ("xray", 1.0, IDENTITY)]
    for calls in (1, 7, n):
        images = run(ctx, trajs, msgs, rows, stages, calls=calls)[3]
        assert images[0].tolist() == [[0xFF000000 | 191 << 16]]


def test_device_buffers_give_the_same_images(ctx):
    import torch
    trajs, msgs, rows = street(num_scans=8, transient_scans=3)
    msgs = with_frames(msgs, (0, 1))
    kw = dict(range_filter=(1.0, 60.0), outlier_voxel_size=0.1)
    host = run(ctx, trajs, msgs, rows, BACKPACK, **kw)
    w = make_writer(ctx, trajs, **kw)
    ids = [i for i in add_stages(w, BACKPACK) if i is not None]
    rows_dev = torch.from_numpy(rows).cuda()
    out_dev = torch.zeros((len(rows), 3), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    while True:
        n, _, _ = w.process_dev(msgs, rows_dev.data_ptr(), len(rows), out_dev.data_ptr())
        if not w.flush():
            break
    ctx.synchronize()
    assert out_dev[:n].cpu().numpy().tobytes() == host[0].tobytes()
    assert_images([w.xray_image(i) for i in ids], host[3])


def test_rejections_leave_the_writer_unchanged(ctx):
    import dliom
    trajs, msgs, rows = street(num_scans=4, transient_scans=0)
    msgs = with_frames(msgs, (0, 1))
    stages = [("color", 0, (10, 20, 30)), ("xray", VOXEL, XY)]
    w = make_writer(ctx, trajs)
    add_stages(w, stages)
    bad_xrays = [(0.0, IDENTITY), (-1.0, IDENTITY), (float("nan"), IDENTITY), (float("inf"), IDENTITY), (1e-50, IDENTITY),
                 (VOXEL, (0, 0, 0, 1.0 + 2e-9, 0, 0, 0)), (VOXEL, (0, 0, 0, 0.6, 0.6, 0, 0)), (VOXEL, (float("nan"),) + IDENTITY[1:])]
    for voxel, transform in bad_xrays:
        with pytest.raises(dliom.DlError) as e:
            w.add_xray(voxel, transform)
        assert e.value.status == -2
    w.add_xray(VOXEL, (0, 0, 0, 1.0 + 0.9e-9, 0, 0, 0))        # within FromDictionary's 1e-9
    with pytest.raises(dliom.DlError):
        w.xray_image(0)                                          # before the final flush
    # a point whose X-ray cell lies beyond +-8192 at 5 cm (the map writer itself takes it: no moving-object removal)
    far = rows.copy()
    far[msgs[1][1] + 3, :3] = (0.0, 0.0, 500.0)
    with pytest.raises(dliom.DlError) as e:
        w.process(msgs, far)
    assert e.value.status == -2 and "X-ray" in str(e.value)
    far_points = mo.write_map(oracle_trajs(trajs), [m[:5] for m in msgs], far)["points"]
    with pytest.raises(ValueError):
        xo.xray_images(far_points, np.zeros(len(far_points)), stages)
    w.process(msgs, rows)
    with pytest.raises(dliom.DlError):
        w.add_color(0, (1, 2, 3))                                # after processing began
    with pytest.raises(dliom.DlError):
        w.add_xray(VOXEL, IDENTITY)
    assert w.flush() is False
    with pytest.raises(dliom.DlError):
        w.xray_image(2)                                          # unknown stage
    with pytest.raises(dliom.DlError):
        w.xray_image(-1)
    res, want = oracle_images(trajs, msgs, rows, stages + [("xray", VOXEL, (0, 0, 0, 1.0 + 0.9e-9, 0, 0, 0))])
    assert_images([w.xray_image(0), w.xray_image(1)], want)
    # the cap on stages, DL_MAP_WRITER_MAX_STAGES = 16 of both kinds together
    c = make_writer(ctx, trajs)
    for k in range(8):
        c.add_color(k, (k, k, k))
        c.add_xray(1.0, IDENTITY)
    with pytest.raises(dliom.DlError):
        c.add_xray(1.0, IDENTITY)
    with pytest.raises(dliom.DlError):
        c.add_color(0, (0, 0, 0))
    # an empty stream: an empty bounding box, a 0 x 0 image
    e = make_writer(ctx, trajs)
    s = e.add_xray(1.0, IDENTITY)
    e.process([], rows)
    e.flush()
    assert e.xray_image(s).shape == (0, 0)


def test_cpp_example_writes_the_same_png_bytes(ctx, tmp_path):
    """build/example_xray (io::MapWriter, ColoringPointsProcessor, XRayPointsProcessor) writes the backpack pipeline's six PNG
    files, byte for byte those of dliom.write_png over dliom.MapWriter on the same input."""
    import dliom
    import __graft_entry__
    from test_map_writer_oracle import write_map_input
    trajs, msgs, rows = street(num_scans=8, transient_scans=3)
    kw = dict(range_filter=(1.0, 40.0), outlier_voxel_size=0.2)
    path = str(tmp_path / "input.bin")
    write_map_input(path, trajs, msgs, rows, range_filter=kw["range_filter"], voxel_size=kw["outlier_voxel_size"])
    r = subprocess.run([__graft_entry__.XRAY_EXAMPLE, path, str(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    pts, _, _, images = run(ctx, trajs, with_frames(msgs, (0, 1)), rows, BACKPACK, **kw)
    names = ["xray_yz_all", "xray_xy_all", "xray_xz_all", "xray_yz_all_color", "xray_xy_all_color", "xray_xz_all_color"]
    lines = r.stdout.split("\n")
    assert lines[0] == f"points {len(pts)}"
    for name, img, line in zip(names, images, lines[1:]):
        assert line == f"{name} {img.shape[1]} {img.shape[0]}"
        assert (tmp_path / (name + ".png")).read_bytes() == dliom.png_bytes(img)
