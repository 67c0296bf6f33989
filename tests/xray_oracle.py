"""CPU oracle of the map writer's X-ray and colour stages (dl_map_writer_add_xray / _add_color / _xray_image), test
infrastructure: the reference's arithmetic restated in numpy, float32 in numpy float32 arrays, double in Python floats (glibc's
log through `math`).

Restated (C/ = cartographer/):
  ColoringPointsProcessor::Process        C/io/coloring_points_processor.cc (last matching stage wins, Uint8ComponentToFloat)
  XRayPointsProcessor::Insert             C/io/xray_points_processor.cc (voxel set, bounding box, float column sums in order)
  XRayPointsProcessor::WriteVoxels        the pixel flip, mean = sum / count in float
  IntoImage / Mix / FloatComponentToUint8 including their promotions: log(size_t) in double, max in float, Mix's a * (1. - t) in
                                          double and t * b in float, Clamp(c) * 255 in float, lround
  Uint8ColorToCairo                       C/io/image.cc
The cell index and the transform reuse map_writer_oracle (hybrid_grid.h:430-435, Eigen's quaternion rotation order).
"""
import math

import numpy as np

import map_writer_oracle as mo

f32 = np.float32
FLT_MIN = float(np.finfo(np.float32).tiny)
WHITE = 0xFFFFFFFF


def point_colors(frames, colors):
    """Colours of a batch's points after the colour stages `colors` [(frame_id, (r, g, b))]: (n, 3) float32, (0, 0, 0)
    (kDefaultColor) where no stage matched."""
    out = np.zeros((len(frames), 3), np.float32)
    for frame, rgb in colors:
        out[np.asarray(frames) == frame] = np.array([f32(int(c) & 0xFF) / f32(255.0) for c in rgb], np.float32)
    return out


def mix(a, b, t):
    """Mix(a, b, t) = a * (1. - t) + t * b: the first product in double, t * b in float, the sum in double, cast to float."""
    return f32(float(a) * (1.0 - float(t)) + float(f32(t) * f32(b)))


def to_uint8(c):
    """FloatComponentToUint8: lround(Clamp(c, 0.f, 1.f) * 255), the product in float."""
    c = min(max(f32(c), f32(0.0)), f32(1.0))
    return int(mo.lround(np.array([f32(c) * f32(255.0)], np.float32))[0]) & 0xFF


def xray_stage(points, frames, voxel_size, transform7, colors):
    """One write_xray_image stage over the stream's points (n, 3) float32 with their frame ids -> the image (height, width)
    uint32 Cairo words. colors: the colour stages added before the stage, in order."""
    pts = np.asarray(points, np.float32).reshape(-1, 3)
    if len(pts) == 0:
        return np.zeros((0, 0), np.uint32)
    pose = np.asarray(transform7, np.float64).astype(np.float32)
    x, y, z = mo.apply_f(pose, pts[:, 0], pts[:, 1], pts[:, 2])
    cx, cy, cz = mo.cell_index(x, y, z, f32(voxel_size))
    if not mo.in_extent(cx, cy, cz).all():
        raise ValueError("an X-ray cell lies beyond the hybrid grid's largest extent")
    col_keys, col_of = np.unique(((cy + mo.GRID_HALF) << 14) | (cz + mo.GRID_HALF), return_inverse=True)
    count = np.bincount(col_of, minlength=len(col_keys)).astype(np.uint32)
    sums = np.zeros((len(col_keys), 3), np.float32)
    np.add.at(sums, col_of, point_colors(frames, colors))     # unbuffered, in stream order: the reference's float additions
    voxel_keys, voxel_first = np.unique(mo.cell_key(cx, cy, cz), return_index=True)
    voxels = np.bincount(col_of[voxel_first], minlength=len(col_keys))
    max_y, min_y, max_z, min_z = int(cy.max()), int(cy.min()), int(cz.max()), int(cz.min())
    width, height = max_y - min_y + 1, max_z - min_z + 1
    img = np.full((height, width), WHITE, np.uint32)
    max_log = f32(FLT_MIN)
    for n in voxels:
        max_log = max(max_log, f32(math.log(int(n))))
    for k, key in enumerate(col_keys.tolist()):
        yy, zz = (key >> 14) - mo.GRID_HALF, (key & 0x3fff) - mo.GRID_HALF
        saturation = f32(math.log(int(voxels[k])) / float(max_log))
        mean = sums[k] / f32(count[k])
        r, g, b = (to_uint8(mix(1.0, mean[c], saturation)) for c in range(3))
        img[max_z - zz, max_y - yy] = 0xFF000000 | r << 16 | g << 8 | b
    return img


def xray_images(points, frames, stages):
    """stages, in pipeline order: ("color", frame_id, rgb) or ("xray", voxel_size, transform7) -> [image per X-ray stage]."""
    colors, images = [], []
    for s in stages:
        if s[0] == "color":
            colors.append((s[1], s[2]))
        else:
            images.append(xray_stage(points, frames, s[1], s[2], list(colors)))
    return images


def final_pass(trajectories, msgs, rows, range_filter=None, voxel_size=0.0):
    """map_writer_oracle.write_map's final-pass points and the frame id of each: msgs [(stamp, first_row, num_rows,
    trajectory_id, sensor_to_tracking7[, frame_id])]. Messages are independent up to the moving-object removal, whose keep
    rule is applied again here from the oracle's cell table."""
    plain = [m[:5] for m in msgs]
    res = mo.write_map(trajectories, plain, rows, range_filter=range_filter, voxel_size=voxel_size)
    per_msg = [mo.write_map(trajectories, [m], rows, range_filter=range_filter)["points"] for m in plain]
    frames = np.concatenate([np.full(len(p), m[5] if len(m) > 5 else 0, np.int64) for m, p in zip(msgs, per_msg)]
                            + [np.zeros(0, np.int64)])
    if voxel_size > 0:
        allpts = np.concatenate([np.zeros((0, 3), np.float32)] + per_msg)
        cx, cy, cz = mo.cell_index(allpts[:, 0], allpts[:, 1], allpts[:, 2], f32(voxel_size))
        table = mo.cell_key(res["cells"][:, 0].astype(np.int64), res["cells"][:, 1].astype(np.int64),
                            res["cells"][:, 2].astype(np.int64))
        pos = np.searchsorted(table, mo.cell_key(cx, cy, cz))
        keep = res["rays"][pos].astype(np.float64) < 3.0 * res["hits"][pos].astype(np.float64)
        assert np.array_equal(allpts[keep], res["points"])
        frames = frames[keep]
    return res, frames
