"""Reference of the map writer's probability-grid stages (dl_map_writer_add_probability_grid / _probability_grid), test
infrastructure: the reference's 2D grid restated literally, float32 in numpy float32 scalars and arrays, double in Python
floats, C's integer arithmetic in Python ints.

Restated (C/ = cartographer/):
  MapLimits::GetCellIndex / Contains          C/mapping/2d/map_limits.h:69-84 (x from y, y from x, lround in double)
  Grid2D::GrowLimits / ComputeCroppedLimits   C/mapping/2d/grid_2d.cc:101-145
  ProbabilityGrid::ApplyLookupTable           C/mapping/2d/probability_grid.cc:53-66 (kUpdateMarker, the known-cells box)
  Grid2D::FinishUpdate                        C/mapping/2d/grid_2d.cc:76-83
  CastRay / GrowAsNeeded / CastRays           C/mapping/internal/2d/ray_casting.cc:29-203
  the correspondence-cost tables              C/mapping/probability_values.cc:27-36, 85-100, probability_values.h
  CreateProbabilityGrid / DrawProbabilityGrid C/io/probability_grid_points_processor.cc:49-54, 127-158
  Image::Rotate90DegreesClockwise             C/io/image.cc:67-76
  WritePgm / WriteYaml and the ROS origin     cartographer_ros/ros_map.cc, ros_map_writing_points_processor.cc:59-80

`Grid.insert` is the literal sequential Insert. `Grid.insert_fast` gives the same grid from sets: the hit cells, and the cells
of every walk from `walk_cells`, a closed form of CastRay per pixel column (pinned to the literal walk in
tests/test_probability_grid_reference.py); it is what the device tests use on whole drives.
"""
import math

import numpy as np

f32 = np.float32
SUBPIXEL = 1000                       # kSubpixelScale
UPDATE_MARKER = 1 << 15               # kUpdateMarker
MIN_PROBABILITY = f32(0.1)
MAX_PROBABILITY = f32(1.0) - MIN_PROBABILITY
MIN_CC = f32(1.0) - MAX_PROBABILITY   # kMinCorrespondenceCost
MAX_CC = f32(1.0) - MIN_PROBABILITY   # kMaxCorrespondenceCost
INITIAL_SIZE = 100                    # kInitialProbabilityGridSize
MAX_CELLS = 100 << 14                 # the superscaled num_cells * 1000 must fit an int
PADDING = f32(1e-6)                   # GrowAsNeeded's kPadding
UNKNOWN_COLOR = 128


def lround(x):
    """std::lround of a double (or a float promoted to double): ties away from zero."""
    a = abs(float(x))
    r = math.floor(a)
    if a - r >= 0.5:
        r += 1
    return int(math.copysign(r, x)) if r else 0


def lround_array(q):
    """lround of a float64 array, exact."""
    a = np.abs(q)
    r = np.floor(a)
    r = r + (a - r >= 0.5)
    return (np.sign(q) * r).astype(np.int64)


def cdiv(a, b):
    """C integer division (truncation toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


# ---- the tables
def value_to_correspondence_cost():
    """kValueToCorrespondenceCost[0, 32768): SlowValueToBoundedFloat(value, 0, kMaxCorrespondenceCost, kMinCC, kMaxCC)."""
    scale = (MAX_CC - MIN_CC) / f32(32766.0)
    out = np.arange(32768).astype(np.float32) * scale + (MIN_CC - scale)
    out[0] = MAX_CC
    return out


def correspondence_cost_to_value(c):
    """CorrespondenceCostToValue of float32 values: RoundToInt((Clamp(c) - lo) * (32766.f / (hi - lo))) + 1."""
    c = np.clip(np.asarray(c, np.float32), MIN_CC, MAX_CC)
    return (lround_array(((c - MIN_CC) * (f32(32766.0) / (MAX_CC - MIN_CC))).astype(np.float64)) + 1).astype(np.int64)


def odds(p):
    p = f32(p)
    return p / (f32(1.0) - p)


def probability_from_odds(o):
    return o / (o + f32(1.0))


def correspondence_cost_table(probability):
    """ComputeLookupTableToApplyCorrespondenceCostOdds(Odds((float)probability)), with the update marker: uint16[32768]."""
    o = odds(probability)
    table = np.zeros(32768, np.int64)
    table[0] = correspondence_cost_to_value(f32(1.0) - probability_from_odds(o)) + UPDATE_MARKER
    p = f32(1.0) - value_to_correspondence_cost()[1:]           # CorrespondenceCostToProbability
    table[1:] = correspondence_cost_to_value(f32(1.0) - probability_from_odds(o * (p / (f32(1.0) - p)))) + UPDATE_MARKER
    return table.astype(np.uint16)


def probability_of(values):
    """ProbabilityGrid::GetProbability of cell values: 1 - kValueToCorrespondenceCost[value], float32 (the table repeats
    itself for values with the update marker)."""
    return f32(1.0) - np.tile(value_to_correspondence_cost(), 2)[np.asarray(values, np.int64)]


def color_table():
    """DrawProbabilityGrid's grey value of every cell value: kUnknownValue 128 for 0, else ProbabilityToColor(GetProbability):
    RoundToInt(255 * ((1.f - p - kMinProbability) / (kMaxProbability - kMinProbability))) in float, as uint8."""
    p = probability_of(np.arange(32768))
    q = f32(1.0) - p
    v = lround_array((f32(255.0) * ((q - MIN_PROBABILITY) / (MAX_PROBABILITY - MIN_PROBABILITY))).astype(np.float64))
    out = (v & 0xFF).astype(np.uint8)
    out[0] = UNKNOWN_COLOR
    return out


# ---- limits
class Limits:
    """MapLimits: resolution and max in double, cell counts."""

    def __init__(self, resolution, max_x, max_y, num_x, num_y):
        self.resolution, self.max_x, self.max_y, self.num_x, self.num_y = float(resolution), float(max_x), float(max_y), num_x, num_y

    def cell_index(self, px, py):
        """GetCellIndex of a float point: (lround((max.y - p.y) / res - 0.5), lround((max.x - p.x) / res - 0.5))."""
        return (lround((self.max_y - float(f32(py))) / self.resolution - 0.5),
                lround((self.max_x - float(f32(px))) / self.resolution - 0.5))

    def contains(self, x, y):
        return 0 <= x < self.num_x and 0 <= y < self.num_y

    def superscaled(self):
        """CastRays' superscaled limits: resolution / kSubpixelScale, the same max, cells * kSubpixelScale."""
        return Limits(self.resolution / SUBPIXEL, self.max_x, self.max_y, self.num_x * SUBPIXEL, self.num_y * SUBPIXEL)

    def cell_indices(self, px, py):
        """cell_index of float32 arrays, vectorized (the same double arithmetic)."""
        return (lround_array((self.max_y - np.asarray(py, np.float32).astype(np.float64)) / self.resolution - 0.5),
                lround_array((self.max_x - np.asarray(px, np.float32).astype(np.float64)) / self.resolution - 0.5))


class GrowthRefused(ValueError):
    """A batch whose growth would pass MAX_CELLS cells per axis."""


def grown_limits(limits, px, py):
    """GrowLimits on the limits alone: the doublings until (px, py)'s cell is contained; GrowthRefused past MAX_CELLS."""
    l = limits
    while not l.contains(*l.cell_index(px, py)):
        if 2 * l.num_x > MAX_CELLS or 2 * l.num_y > MAX_CELLS:
            raise GrowthRefused("growth beyond %d cells per axis" % MAX_CELLS)
        l = Limits(l.resolution, l.max_x + l.resolution * float(l.num_y // 2), l.max_y + l.resolution * float(l.num_x // 2),
                   2 * l.num_x, 2 * l.num_y)
    return l


class Grid:
    """ProbabilityGrid with its known-cells box and update list; cells[y, x] uint16 (flat index num_x * y + x)."""

    def __init__(self, resolution):
        """CreateProbabilityGrid(resolution): 100 x 100 cells, max = 0.5 * 100 * resolution per axis."""
        m = 0.5 * INITIAL_SIZE * float(resolution)
        self.limits = Limits(resolution, m, m, INITIAL_SIZE, INITIAL_SIZE)
        self.cells = np.zeros((INITIAL_SIZE, INITIAL_SIZE), np.uint16)
        self.box = None                  # [min_x, min_y, max_x, max_y] or None (empty)
        self.update = []

    @classmethod
    def from_limits(cls, limits):
        """ProbabilityGrid(MapLimits): every cell unknown."""
        g = cls.__new__(cls)
        g.limits = limits
        g.cells = np.zeros((limits.num_y, limits.num_x), np.uint16)
        g.box, g.update = None, []
        return g

    def set_probability(self, x, y, probability):
        """ProbabilityGrid::SetProbability: only on an unknown cell."""
        assert self.cells[y, x] == 0
        self.cells[y, x] = correspondence_cost_to_value(f32(1.0) - f32(probability))
        self.extend_box(x, y, x, y)

    def is_known(self, x, y):
        return self.limits.contains(x, y) and self.cells[y, x] != 0

    def get_probability(self, x, y):
        if not self.limits.contains(x, y):
            return MIN_PROBABILITY
        return probability_of(self.cells[y, x])

    # Grid2D::GrowLimits
    def grow_limits(self, px, py):
        assert not self.update
        while not self.limits.contains(*self.limits.cell_index(px, py)):
            l = self.limits
            if 2 * l.num_x > MAX_CELLS or 2 * l.num_y > MAX_CELLS:
                raise GrowthRefused("growth beyond %d cells per axis" % MAX_CELLS)
            x_offset, y_offset = l.num_x // 2, l.num_y // 2
            new = Limits(l.resolution, l.max_x + l.resolution * float(y_offset), l.max_y + l.resolution * float(x_offset),
                         2 * l.num_x, 2 * l.num_y)
            cells = np.zeros((new.num_y, new.num_x), np.uint16)
            cells[y_offset:y_offset + l.num_y, x_offset:x_offset + l.num_x] = self.cells
            self.cells, self.limits = cells, new
            if self.box is not None:
                self.box = [self.box[0] + x_offset, self.box[1] + y_offset, self.box[2] + x_offset, self.box[3] + y_offset]

    # ProbabilityGrid::ApplyLookupTable
    def apply_lookup_table(self, x, y, table):
        if not self.limits.contains(x, y):
            raise IndexError("ToFlatIndex CHECK: cell (%d, %d) outside the limits" % (x, y))
        if self.cells[y, x] >= UPDATE_MARKER:
            return False
        self.update.append((x, y))
        self.cells[y, x] = table[self.cells[y, x]]
        self.extend_box(x, y, x, y)
        return True

    def extend_box(self, x0, y0, x1, y1):
        b = self.box
        self.box = [x0, y0, x1, y1] if b is None else [min(b[0], x0), min(b[1], y0), max(b[2], x1), max(b[3], y1)]

    def finish_update(self):
        for x, y in self.update:
            assert self.cells[y, x] >= UPDATE_MARKER
            self.cells[y, x] -= UPDATE_MARKER
        self.update = []

    def grow_as_needed(self, origin, points):
        """The float AlignedBox2f of the origin and the points' x y, then GrowLimits(min - 1e-6f), GrowLimits(max + 1e-6f)."""
        xy = np.vstack([np.asarray(origin, np.float32).reshape(1, -1)[:, :2], np.asarray(points, np.float32).reshape(-1, 3)[:, :2]
                        if len(points) else np.zeros((0, 2), np.float32)])
        lo, hi = xy.min(axis=0), xy.max(axis=0)
        grown_limits(grown_limits(self.limits, lo[0] - PADDING, lo[1] - PADDING), hi[0] + PADDING, hi[1] + PADDING)  # refuse first
        self.grow_limits(lo[0] - PADDING, lo[1] - PADDING)
        self.grow_limits(hi[0] + PADDING, hi[1] + PADDING)

    def insert(self, origin, points, hit_table, miss_table, insert_free_space=True):
        """ProbabilityGridRangeDataInserter2D::Insert({origin, points, {}}): CastRays, then FinishUpdate."""
        self.grow_as_needed(origin, points)
        ss = self.limits.superscaled()
        begin = ss.cell_index(origin[0], origin[1])
        ends = [ss.cell_index(p[0], p[1]) for p in np.asarray(points, np.float32).reshape(-1, 3)]
        for e in ends:
            self.apply_lookup_table(cdiv(e[0], SUBPIXEL), cdiv(e[1], SUBPIXEL), hit_table)
        if insert_free_space:
            for e in ends:
                cast_ray(begin, e, lambda x, y: self.apply_lookup_table(x, y, miss_table))
        self.finish_update()

    def insert_fast(self, origin, points, hit_table, miss_table, insert_free_space=True):
        """The same grid as insert() from sets: every hit cell gets the hit table once, every other walked cell the miss table
        once."""
        self.grow_as_needed(origin, points)
        pts = np.asarray(points, np.float32).reshape(-1, 3)
        if len(pts) == 0:
            return
        ss = self.limits.superscaled()
        bx, by = ss.cell_index(origin[0], origin[1])
        ex, ey = ss.cell_indices(pts[:, 0], pts[:, 1])
        nx = self.limits.num_x
        hits = np.unique((ey // SUBPIXEL) * nx + ex // SUBPIXEL)
        flat = self.cells.reshape(-1)
        changed = [hits]
        if insert_free_space:
            cx, cy = walk_cells(bx, by, ex, ey)
            if ((cx < 0) | (cy < 0) | (cx >= nx) | (cy >= self.limits.num_y)).any():
                raise IndexError("a walk leaves the limits")
            misses = np.setdiff1d(np.unique(cy * nx + cx), hits)
            flat[misses] = miss_table[flat[misses]] - UPDATE_MARKER
            changed.append(misses)
        flat[hits] = hit_table[flat[hits]] - UPDATE_MARKER
        idx = np.concatenate(changed)
        self.extend_box(int((idx % nx).min()), int((idx // nx).min()), int((idx % nx).max()), int((idx // nx).max()))

    # ComputeCroppedLimits
    def cropped(self):
        """(offset_x, offset_y, width, height): the known-cells box, or (0, 0, 1, 1) when it is empty."""
        if self.box is None:
            return 0, 0, 1, 1
        return self.box[0], self.box[1], self.box[2] - self.box[0] + 1, self.box[3] - self.box[1] + 1

    def cropped_cells(self):
        ox, oy, w, h = self.cropped()
        return self.cells[oy:oy + h, ox:ox + w]

    def image(self):
        """DrawProbabilityGrid: (height, width) uint8 grey values of the cropped box, pixel (x, y) = cell (x, y) + offset."""
        return color_table()[self.cropped_cells().astype(np.int64)]

    def info(self):
        l = self.limits
        ox, oy, w, h = self.cropped()
        return {"resolution": l.resolution, "max_x": l.max_x, "max_y": l.max_y, "num_x_cells": l.num_x, "num_y_cells": l.num_y,
                "offset_x": ox, "offset_y": oy, "width": w, "height": h}


def xy_index_range(lo, hi):
    """XYIndexRangeIterator(min, max): x fastest, both bounds inclusive."""
    for y in range(lo[1], hi[1] + 1):
        for x in range(lo[0], hi[0] + 1):
            yield x, y


def cast_ray(begin, end, visit):
    """CastRay (ray_casting.cc:29-146), literally: visit(x, y) for every full pixel, in the reference's order."""
    if begin[0] > end[0]:
        cast_ray(end, begin, visit)
        return
    assert begin[0] >= 0 and begin[1] >= 0 and end[1] >= 0
    S = SUBPIXEL
    if begin[0] // S == end[0] // S:
        x = begin[0] // S
        for y in range(min(begin[1], end[1]) // S, max(begin[1], end[1]) // S + 1):
            visit(x, y)
        return
    dx, dy = end[0] - begin[0], end[1] - begin[1]
    denominator = 2 * S * dx
    cx, cy = begin[0] // S, begin[1] // S
    sub_y = (2 * (begin[1] % S) + 1) * dx
    first_pixel = 2 * S - 2 * (begin[0] % S) - 1
    last_pixel = 2 * (end[0] % S) + 1
    end_x = max(begin[0], end[0]) // S
    sub_y += dy * first_pixel
    if dy > 0:
        while True:
            visit(cx, cy)
            while sub_y > denominator:
                sub_y -= denominator
                cy += 1
                visit(cx, cy)
            cx += 1
            if sub_y == denominator:
                sub_y -= denominator
                cy += 1
            if cx == end_x:
                break
            sub_y += dy * 2 * S
        sub_y += dy * last_pixel
        visit(cx, cy)
        while sub_y > denominator:
            sub_y -= denominator
            cy += 1
            visit(cx, cy)
        assert sub_y != denominator and cy == end[1] // S
        return
    while True:
        visit(cx, cy)
        while sub_y < 0:
            sub_y += denominator
            cy -= 1
            visit(cx, cy)
        cx += 1
        if sub_y == 0:
            sub_y += denominator
            cy -= 1
        if cx == end_x:
            break
        sub_y += dy * 2 * S
    sub_y += dy * last_pixel
    visit(cx, cy)
    while sub_y < 0:
        sub_y += denominator
        cy -= 1
        visit(cx, cy)
    assert sub_y != 0 and cy == end[1] // S


def walk_cells(bx, by, ex, ey):
    """The pixels of CastRay((bx, by), (ex[i], ey[i])) for every i, as (x, y) int64 arrays (with repeats across walks). Per
    pixel column the walk covers a closed range of rows: with T the unreduced sub_y at the column's right border (the last
    column adds dy * last_pixel instead of dy * 2S), D = 2S * dx, a rising walk leaves column j at row y0 + ceil(T/D) - 1 and
    enters column j + 1 at y0 + floor(T/D) (the corner rule); a non-rising one leaves at y0 - max(0, ceil(-T/D)) and enters
    at y0 - floor(-T/D) - 1."""
    S = SUBPIXEL
    ex, ey = np.asarray(ex, np.int64), np.asarray(ey, np.int64)
    b0x, b0y = np.full_like(ex, bx), np.full_like(ey, by)
    swap = b0x > ex
    x0, y0, x1, y1 = np.where(swap, ex, b0x), np.where(swap, ey, b0y), np.where(swap, b0x, ex), np.where(swap, b0y, ey)
    out_x, out_y = [], []
    vertical = x0 // S == x1 // S
    if vertical.any():
        lo, hi = np.minimum(y0, y1)[vertical] // S, np.maximum(y0, y1)[vertical] // S
        n = hi - lo + 1
        walk = np.repeat(np.arange(len(n)), n)
        out_x.append(np.repeat((x0[vertical] // S), n))
        out_y.append(lo[walk] + (np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n)))
    k = ~vertical
    if k.any():
        x0, y0, x1, y1 = x0[k], y0[k], x1[k], y1[k]
        dx, dy = x1 - x0, y1 - y0
        D = 2 * S * dx
        m = x1 // S - x0 // S                     # columns before the last one
        t0 = (2 * (y0 % S) + 1) * dx + dy * (2 * S - 2 * (x0 % S) - 1)
        cols = m + 1
        walk = np.repeat(np.arange(len(m)), cols)
        j = np.arange(cols.sum()) - np.repeat(np.cumsum(cols) - cols, cols)
        last = j == m[walk]
        T = t0[walk] + np.where(last, (j - 1) * 2 * S * dy[walk] + dy[walk] * (2 * (x1[walk] % S) + 1),
                                j * 2 * S * dy[walk])
        Tprev = t0[walk] + (j - 1) * 2 * S * dy[walk]     # the previous column's T (j >= 1)
        Dw, yb, up = D[walk], (y0 // S)[walk], dy[walk] > 0
        ceil_div = lambda a, b: -((-a) // b)
        # the row a column is entered at and left at
        enter_up = np.where(j == 0, yb, yb + Tprev // Dw)
        leave_up = yb + ceil_div(T, Dw) - 1
        enter_down = np.where(j == 0, yb, yb - (-Tprev) // Dw - 1)
        leave_down = yb - np.maximum(0, ceil_div(-T, Dw))
        a = np.where(up, enter_up, leave_down)
        b = np.where(up, leave_up, enter_down)
        n = b - a + 1
        assert (n >= 1).all()
        cx = (x0 // S)[walk] + j
        out_x.append(np.repeat(cx, n))
        out_y.append(np.repeat(a, n) + (np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n)))
    if not out_x:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(out_x), np.concatenate(out_y)


def rotate90_clockwise(image):
    """Image::Rotate90DegreesClockwise: new row x is old column x read from the bottom row up."""
    img = np.asarray(image)
    h, w = img.shape
    out = np.empty((w, h), img.dtype)
    for x in range(w):
        out[x] = img[::-1, x]
    return out


def pgm_bytes(image, resolution):
    """WritePgm of the rotated image: the header with std::to_string(resolution) (%f), then the red channel row by row."""
    img = np.asarray(image, np.uint8)
    header = "P5\n# Cartographer map; " + ("%f" % resolution) + " m/pixel\n" + "%d %d" % (img.shape[1], img.shape[0]) + "\n255\n"
    return header.encode() + img.tobytes()


def yaml_bytes(resolution, origin, pgm_filename):
    """WriteYaml: map_saver's constants, std::to_string (%f) of the resolution and the origin."""
    return ("image: " + pgm_filename + "\n" + "resolution: " + ("%f" % resolution) + "\n" + "origin: [" + ("%f" % origin[0]) +
            ", " + ("%f" % origin[1]) + ", 0.0]\nnegate: 0\noccupied_thresh: 0.65\nfree_thresh: 0.196\n").encode()


def ros_map(grid_info, image, pgm_filename):
    """RosMapWritingPointsProcessor::Flush: rotate, PGM, and the YAML with origin = (max.x - (offset.y + width) * res,
    max.y - (offset.x + height) * res), width and height after the rotation -> (pgm bytes, yaml bytes)."""
    rotated = rotate90_clockwise(image)
    h, w = rotated.shape
    res = grid_info["resolution"]
    origin = (grid_info["max_x"] - (grid_info["offset_y"] + w) * res, grid_info["max_y"] - (grid_info["offset_x"] + h) * res)
    return pgm_bytes(rotated, res), yaml_bytes(res, origin, pgm_filename)


def run_batches(resolution, hit, miss, batches, insert_free_space=True, fast=True):
    """A grid stage over batches [(origin xyz, points (n, 3) float32)] in order -> the Grid."""
    g = Grid(resolution)
    ht, mt = correspondence_cost_table(hit), correspondence_cost_table(miss)
    for origin, points in batches:
        (g.insert_fast if fast else g.insert)(origin, points, ht, mt, insert_free_space)
    return g
