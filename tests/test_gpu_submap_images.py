"""dl_submap_textures / dl_submap_projections: every byte, size, slice pose and origin equals tests/submap_image_reference.py, a
float32 numpy reading of AddToTextureProto and ProjectToCvMat that takes the cells from dl_grid_export_cells and orders them itself
from the cell index alone."""
import numpy as np
import pytest

import submap_image_reference as ref

RNG_SEED = 11


def rot_pose(t, yaw, roll=0.0, pitch=0.0):
    """7-vector of Rz(yaw) Ry(pitch) Rx(roll) at t (w x y z last four)."""
    cy, sy = np.cos(yaw / 2), np.sin(yaw / 2)
    cp, sp = np.cos(pitch / 2), np.sin(pitch / 2)
    cr, sr = np.cos(roll / 2), np.sin(roll / 2)
    q = [cy * cp * cr + sy * sp * sr, cy * cp * sr - sy * sp * cr, cy * sp * cr + sy * cp * sr, sy * cp * cr - cy * sp * sr]
    return np.array([*t, *q], np.float64)


POSES = [np.array([0, 0, 0, 1, 0, 0, 0], np.float64), rot_pose((3.7, -12.25, 1.5), 0.7),
         rot_pose((-40.0, 8.0, -2.0), -2.3, roll=0.08, pitch=-0.05), rot_pose((0.1, 0.2, 0.3), 3.1, roll=-0.3, pitch=0.25)]


def compose(a, b):
    """a * b of two 7-vector poses (float64; any global pose will do)."""
    def quat_mul(p, q):
        w1, x1, y1, z1 = p
        w2, x2, y2, z2 = q
        return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                         w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])
    v = quat_mul(quat_mul(a[3:], np.r_[0.0, b[:3]]), a[3:] * [1, -1, -1, -1])[1:]
    q = quat_mul(a[3:], b[3:])
    return np.r_[v + a[:3], q / np.linalg.norm(q)]


def assert_texture(got, want):
    assert (got["width"], got["height"]) == (want["width"], want["height"])
    assert np.float32(got["resolution"]) == want["resolution"]
    assert np.array_equal(got["slice_pose"].view(np.uint64), want["slice_pose"].view(np.uint64)), (got["slice_pose"], want["slice_pose"])
    assert np.array_equal(got["cells"], want["cells"])


def assert_projection(got, want):
    assert (got["width"], got["height"]) == (want["width"], want["height"])
    assert np.float32(got["resolution"]) == want["resolution"]
    assert got["ox"] == want["ox"] and got["oy"] == want["oy"]
    assert np.array_equal(got["pixels"], want["pixels"])


def check_grid(ctx, grid, poses, resolution):
    """Textures and projections of `grid` at every pose, one call each, against the reference."""
    cells = grid.export()
    tex = ctx.submap_textures([(grid, p) for p in poses])
    proj = ctx.project_submaps([(grid, p) for p in poses])
    for p, t, j in zip(poses, tex, proj):
        assert_texture(t, ref.texture(*cells, resolution, p))
        assert_projection(j, ref.projection(*cells, resolution, p))
    return tex, proj


def column_grid(ctx, res, rng, n_cols=300, spread=80, base=(0, 0, 0)):
    """Columns of cells (z runs of several lengths) so that textures have pixels on both sides of z_difference 3, across 64- and
    8-cell boundaries, with every probability band."""
    import dliom
    xs, ys, zs, vs = [], [], [], []
    for _ in range(n_cols):
        x, y = rng.integers(-spread, spread, 2) + np.array(base[:2])
        z0 = int(rng.integers(-70, 70)) + base[2]
        for dz in range(int(rng.integers(1, 12))):
            xs.append(x); ys.append(y); zs.append(z0 + dz * int(rng.integers(1, 4)))
            vs.append(int(rng.choice([rng.integers(1, 32768), rng.integers(16000, 16500), 32767, 1])))
    g = dliom.Grid(ctx, res)
    xyz = np.clip(np.stack([xs, ys, zs], 1), -8192, 8191)  # the grid's range at bits 8
    xyz, first = np.unique(xyz, axis=0, return_index=True)
    g.set_cells(xyz[:, 0], xyz[:, 1], xyz[:, 2], np.asarray(vs)[first])
    return g


@pytest.mark.gpu
def test_hand_placed_grids_all_poses():
    import dliom
    ctx = dliom.Context(0)
    rng = np.random.default_rng(RNG_SEED)
    for res in (0.2, 0.45, 0.1):
        check_grid(ctx, column_grid(ctx, np.float32(res), rng), POSES, np.float32(res))


@pytest.mark.gpu
def test_pixel_sums_follow_iterator_order(monkeypatch):
    """Cells inserted top down, so that the brick pool's order is not the iterator's; the values make the output byte differ
    under the reverse summation order (tests/test_submap_image_reference.py)."""
    import dliom
    import test_submap_image_reference as cases
    ctx = dliom.Context(0)
    for resolution in (np.float32(1.0), np.float32(0.2)):
        for values in (cases.ORDER_PROJECTION_VALUES, cases.ORDER_TEXTURE_VALUES):
            xs, ys, zs, vs = cases.order_case(values)
            g = dliom.Grid(ctx, resolution)
            g.set_cells(xs, ys, zs, vs)
            tex, proj = check_grid(ctx, g, POSES[:1], resolution)
            with monkeypatch.context() as m:
                m.setattr(ref, "iterator_order", cases.reversed_iterator_order)
                wrong_tex = ref.texture(*g.export(), resolution, POSES[0])
                wrong_proj = ref.projection(*g.export(), resolution, POSES[0])
            if values is cases.ORDER_TEXTURE_VALUES:
                assert not np.array_equal(tex[0]["cells"], wrong_tex["cells"])
            else:
                assert not np.array_equal(proj[0]["pixels"], wrong_proj["pixels"])


@pytest.mark.gpu
def test_cells_near_the_grid_limit_and_grown_grids_keep_iterator_order():
    """Cells near +-8192 grow the grid to bits 8; the export's order (the Iterator's) must equal the reference's ordering."""
    import dliom
    ctx = dliom.Context(0)
    rng = np.random.default_rng(RNG_SEED + 1)
    for base in ((8150, -8150, 8140), (-8180, 8170, -8100), (300, -700, 40)):
        g = column_grid(ctx, np.float32(0.2), rng, n_cols=120, spread=60, base=base)
        xs, ys, zs, _ = g.export()
        assert np.array_equal(ref.iterator_order(xs, ys, zs), np.arange(len(xs)))
        check_grid(ctx, g, POSES, np.float32(0.2))
    # growing step by step: every stage in iterator order and equal to the reference
    g = dliom.Grid(ctx, 0.3)
    for k, reach in enumerate((50, 200, 900, 3000, 8000)):
        pts = rng.integers(-reach, reach, (200, 3))
        g.set_cells(pts[:, 0], pts[:, 1], pts[:, 2] // 8, rng.integers(16384, 32768, 200))
        xs, ys, zs, _ = g.export()
        assert np.array_equal(ref.iterator_order(xs, ys, zs), np.arange(len(xs))), k
        check_grid(ctx, g, POSES[:2], np.float32(0.3))


@pytest.mark.gpu
def test_empty_and_unobstructed_grids_give_0_by_0():
    import dliom
    ctx = dliom.Context(0)
    empty = dliom.Grid(ctx, 0.2)
    empty.sync()
    free = dliom.Grid(ctx, 0.2)
    free.set_cells([0, 5, -3], [1, 2, 3], [0, 0, 9], [100, 16400, 16000])  # every probability below 0.501
    full = column_grid(ctx, np.float32(0.2), np.random.default_rng(3), n_cols=20)
    tex = ctx.submap_textures([(empty, POSES[1]), (free, POSES[1]), (full, POSES[1])])
    proj = ctx.project_submaps([(empty, POSES[1]), (free, POSES[1]), (full, POSES[1])])
    for t, j in zip(tex[:2], proj[:2]):
        assert (t["width"], t["height"], j["width"], j["height"]) == (0, 0, 0, 0)
        assert not t["slice_pose"].any() and j["ox"] == 0.0 and j["oy"] == 0.0
    assert_texture(tex[2], ref.texture(*full.export(), np.float32(0.2), POSES[1]))
    assert_projection(proj[2], ref.projection(*full.export(), np.float32(0.2), POSES[1]))


@pytest.mark.gpu
def test_32_queries_equal_32_single_calls_with_constant_launches():
    import dliom
    ctx = dliom.Context(0)
    rng = np.random.default_rng(RNG_SEED + 2)
    grids = [column_grid(ctx, np.float32(r), rng, n_cols=60) for r in (0.2, 0.45, 0.2, 0.1)]
    queries = [(grids[k % 4], rot_pose(rng.normal(0, 5, 3), rng.uniform(-3, 3), *rng.normal(0, 0.1, 2))) for k in range(32)]
    for fn in (ctx.submap_textures, ctx.project_submaps):
        before = ctx.launches
        many = fn(queries)
        launches_many = ctx.launches - before
        before = ctx.launches
        one = fn(queries[:1])
        launches_one = ctx.launches - before
        assert launches_many == launches_one
        for q, m in zip(queries, many):
            s = fn([q])[0]
            for key in m:
                assert np.array_equal(np.asarray(m[key]), np.asarray(s[key])), key


@pytest.mark.gpu
def test_queries_follow_device_insertion_and_leave_the_grid_unchanged():
    import dliom
    ctx = dliom.Context(0)
    rng = np.random.default_rng(RNG_SEED + 3)
    g = dliom.Grid(ctx, 0.2)
    g.sync()
    origin = np.zeros(3, np.float32)
    for k in range(6):
        pts = (rng.normal(0, 1, (3000, 3)) * [12, 12, 2] + [0, 0, 1]).astype(np.float32)
        g.insert_range_data(origin, pts)
        before = g.export()
        tex, proj = check_grid(ctx, g, POSES[:3], np.float32(0.2))
        after = g.export()
        assert all(np.array_equal(a, b) for a, b in zip(before, after))
        assert tex[0]["width"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("beams", [16, 64])
def test_every_submap_of_a_drive(orc, beams):
    """dl_ltb's grids (active and finished, both resolutions) at their local poses and at a global correction of them."""
    import dliom
    import synth
    import imu_synth
    import test_gpu_ltb_batch as drive
    ctx = dliom.Context(0)
    tr = drive.Trajectory(synth.Scene(42), 2.0, beams=beams)
    b = dliom.LocalTrajectoryBuilder(ctx, drive.make_options(orc, num_range_data=4, high_resolution=0.2))
    b.set_initial_state(imu_synth.state(tr.t0 - 0.1))
    for _ in range(14):
        t1, imu, xyzt = tr.next()
        drive.feed_imu(b, imu)
        drive.single(b, t1, xyzt)
    assert b.num_submaps() >= 3
    correction = rot_pose((1.5, -2.0, 0.3), 0.4, roll=0.01, pitch=-0.02)
    for i in range(b.num_submaps()):
        hi, lo, local, _, _ = b.submap(i)
        for grid, res in ((hi, np.float32(0.2)), (lo, np.float32(b.options.low_resolution))):
            check_grid(ctx, grid, [local, compose(correction, local)], res)
    b.close()


def build_example(out_dir):
    """host/example_submap_images.cc (the C++ shim's GetSubmap / ToResponseProto / ProjectToCvMat) built with -Wall -Werror."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(str(out_dir), "example_submap_images")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", os.path.join(root, "d-liom_b200", "host", "example_submap_images.cc"),
                           "-o", exe, "-L" + os.path.join(root, "d-liom_b200"), "-ldliom_b200",
                           "-Wl,-rpath," + os.path.join(root, "d-liom_b200")])
    return exe


def pgm(width, height, data):
    return b"P5\n%d %d\n255\n" % (width, height) + bytes(np.ascontiguousarray(data, np.uint8).ravel())


@pytest.mark.gpu
def test_cpp_example_pgms_equal_python_and_pose_graph_poses_equal_the_reference(orc, tmp_path):
    """The C++ example replays a two-trajectory drive through LocalTrajectoryBuilder3D and PoseGraph3D and writes every submap's
    textures (at the pose graph's global submap poses) and projection as PGM files; the same drive replayed from Python, with the
    poses the example printed, must give the same files byte for byte, and the textures at those global poses equal the reference."""
    import struct
    import subprocess
    import dliom
    import imu_synth
    import synth
    import test_gpu_ltb_batch as drive
    exe = build_example(tmp_path)
    trajs = [drive.Trajectory(synth.Scene(42), 2.0 + 0.6 * j) for j in range(2)]
    steps = 10
    inputs = [[tr.next() for tr in trajs] for _ in range(steps)]
    path = str(tmp_path / "drives.bin")
    with open(path, "wb") as f:
        f.write(struct.pack("<i", len(trajs)))
        for tr in trajs:
            f.write(dliom.NavState.from16(imu_synth.state(tr.t0 - 0.1)))
        f.write(struct.pack("<i", steps))
        for row in inputs:
            for t1, imu, xyzt in row:
                f.write(struct.pack("<i", len(imu)))
                for t, a, g in imu:
                    f.write(struct.pack("<d", t) + np.asarray(a, np.float64).tobytes() + np.asarray(g, np.float64).tobytes())
                f.write(struct.pack("<di", t1, len(xyzt)) + xyzt.tobytes())
    out_dir = tmp_path / "pgm"
    out_dir.mkdir()
    r = subprocess.run([exe, path, str(out_dir)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [l.split() for l in r.stdout.splitlines() if l.startswith("submap")]
    assert len(lines) >= 6
    # the same drive from Python
    ctx = dliom.Context(0)
    builders = []
    for tr in trajs:
        b = dliom.LocalTrajectoryBuilder(ctx, drive.make_options(orc, num_range_data=3))
        b.set_initial_state(imu_synth.state(tr.t0 - 0.1))
        builders.append(b)
    for row in inputs:
        for b, (t1, imu, xyzt) in zip(builders, row):
            drive.feed_imu(b, imu)
            drive.single(b, t1, xyzt)
    tex_q, proj_q, names, moved = [], [], [], False
    for l in lines:
        j, i, version = int(l[1]), int(l[2]), int(l[3])
        global_pose = np.array([float(v) for v in l[4:11]])
        local_pose = np.array([float(v) for v in l[11:18]])
        hi, lo, local, n, _ = builders[j].submap(i)
        assert np.array_equal(local.view(np.uint64), local_pose.view(np.uint64)) and n == version, (j, i)
        moved |= not np.array_equal(global_pose, local_pose)
        tex_q += [(hi, global_pose), (lo, global_pose)]
        proj_q.append((hi, local_pose))
        names.append(f"t{j}_s{i}")
    assert moved  # the pose graph's optimization moved some submap away from its local pose
    tex = ctx.submap_textures(tex_q)
    proj = ctx.project_submaps(proj_q)
    for k, name in enumerate(names):
        for t in range(2):
            got = tex[2 * k + t]
            for c, suffix in ((0, "value"), (1, "alpha")):
                want = pgm(got["width"], got["height"], got["cells"][..., c])
                assert (out_dir / f"{name}_tex{t}_{suffix}.pgm").read_bytes() == want, (name, t, suffix)
        p = proj[k]
        assert (out_dir / f"{name}_projection.pgm").read_bytes() == pgm(p["width"], p["height"], p["pixels"]), name
    for (grid, pose), got, res in zip(tex_q, tex, [np.float32(0.1), np.float32(0.45)] * len(names)):
        assert_texture(got, ref.texture(*grid.export(), res, pose))
    for b in builders:
        b.close()
