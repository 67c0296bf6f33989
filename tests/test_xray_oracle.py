"""CPU checks of the X-ray and colour stages: the oracle (tests/xray_oracle.py) on hand-worked cases, RollPitchYaw of
transform.lua's transforms, the PNG writer decoded with zlib, the C++ shim's PNG bytes against dliom.png_bytes, and the C-ABI's
layouts and argument checks."""
import ctypes
import math
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

import xray_oracle as xo

f32 = np.float32
IDENTITY = (0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)
BLACK, WHITE = 0xFF000000, 0xFFFFFFFF
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def pts(*rows):
    return np.array(rows, np.float32).reshape(-1, 3)


def test_pixel_flip_and_image_size():
    # cells (x, y, z) at voxel 1: columns (y, z) = (0, 0), (2, 1) twice (x = 0 and 1: two voxels), (-1, 3)
    p = pts((0, 0, 0), (0, 2, 1), (1, 2, 1), (5, -1, 3))
    img = xo.xray_stage(p, np.zeros(4), 1.0, IDENTITY, [])
    assert img.shape == (4, 4)                       # height = 3 - 0 + 1, width = 2 - (-1) + 1
    want = np.full((4, 4), WHITE, np.uint32)
    want[3 - 1, 2 - 2] = BLACK                       # (max.y - y, max.z - z): saturation log 2 / log 2 = 1, mean colour 0
    assert img.tolist() == want.tolist()             # the single-voxel columns: saturation 0, white like the empty ones


def test_all_single_voxel_columns_render_white():
    p = pts((0, 0, 0), (0, 1, 0), (3, 2, 5), (-4, -1, 1))
    img = xo.xray_stage(p, np.zeros(4), 1.0, IDENTITY, [])
    assert img.shape == (6, 4) and (img == WHITE).all()      # max = FLT_MIN, log(1) / FLT_MIN = 0


def test_color_rule_order_and_frame_matching():
    # three columns of two voxels each (every saturation 1: pixel = mean colour), one per frame id 0, 1, 2
    p = pts((0, 0, 0), (1, 0, 0), (0, 1, 0), (1, 1, 0), (0, 2, 0), (1, 2, 0))
    frames = np.array([0, 0, 1, 1, 2, 2])
    stages = [("color", 0, (255, 0, 0)), ("xray", 1.0, IDENTITY), ("color", 0, (0, 255, 0)), ("color", 1, (0, 0, 255.9)),
              ("xray", 1.0, IDENTITY)]
    a, b = xo.xray_images(p, frames, stages)
    # pixel x = max.y - y
    assert a[0].tolist() == [BLACK, BLACK, 0xFFFF0000]                   # frame 2, frame 1: default colour; frame 0 red
    assert b[0].tolist() == [BLACK, 0xFF0000FF, 0xFF00FF00]              # the last matching stage wins; 255.9 -> 255
    assert xo.xray_images(p, frames, [("xray", 1.0, IDENTITY)])[0][0].tolist() == [BLACK] * 3


def test_mix_takes_the_double_evaluation():
    t, b = np.uint32(1053270447).view(np.float32), np.uint32(1042548175).view(np.float32)
    as_float = f32(f32(f32(1.0) * f32(f32(1.0) - t)) + f32(t * b))        # the same expression all in float
    assert xo.to_uint8(xo.mix(1.0, b, t)) == 172 and xo.to_uint8(as_float) == 171


def test_interleaved_column_sum_depends_on_order():
    # 774 points in one column, two voxels, frames alternating red 255 / 128: the in-order float sum and the sorted one differ
    # by more than a byte of the mean
    n = 774
    p = np.zeros((n, 3), np.float32)
    p[1::2, 0] = 1.0
    frames = np.arange(n) % 2
    colors = [("color", 0, (255, 0, 0)), ("color", 1, (128, 0, 0))]
    img = xo.xray_images(p, frames, colors + [("xray", 1.0, IDENTITY)])[0]
    c = xo.point_colors(frames, [(0, (255, 0, 0)), (1, (128, 0, 0))])[:, 0]
    in_order, reordered = f32(0.0), f32(0.0)
    for v in c:
        in_order = f32(in_order + v)
    for v in np.sort(c):
        reordered = f32(reordered + v)
    assert in_order != reordered
    assert xo.to_uint8(in_order / f32(n)) == 191 and xo.to_uint8(reordered / f32(n)) == 192
    assert img.tolist() == [[0xFF000000 | 191 << 16]]


def test_transform_and_cell_rounding():
    # XY_TRANSFORM looks down the map's z axis: the camera's (y, z) are the map's (y, x) up to sign
    import dliom
    xy = (0.0, 0.0, 0.0) + dliom.roll_pitch_yaw(0.0, -math.pi / 2, 0.0)
    p = pts((2.0, 1.0, 7.0), (2.0, 1.0, -3.0), (-1.0, 0.0, 0.0))
    img = xo.xray_stage(p, np.zeros(3), 1.0, xy, [])
    assert img.shape == (4, 2)                         # y in {0, 1}, camera z = map x in {-1, 2}
    assert (img != WHITE).sum() == 1                   # the column of the two stacked points, the other single-voxel column white
    assert img[0, 0] == BLACK
    half = pts((0.5, -0.5, 1.5), (-2.5, 0.49999997, 0.0))
    cx, cy, cz = xo.mo.cell_index(half[:, 0], half[:, 1], half[:, 2], f32(1.0))
    assert cx.tolist() == [1, -3] and cy.tolist() == [-1, 0] and cz.tolist() == [2, 0]     # lround: ties away from zero


def test_roll_pitch_yaw_of_the_transform_lua_transforms():
    import dliom
    s = math.sqrt(0.5)
    want = {"XY": (s, 0.0, -s, 0.0), "XZ": (s, 0.0, 0.0, -s), "YZ": (0.0, 0.0, 0.0, 1.0)}
    got = {"XY": dliom.roll_pitch_yaw(0.0, -math.pi / 2.0, 0.0), "XZ": dliom.roll_pitch_yaw(0.0, 0.0, -math.pi / 2),
           "YZ": dliom.roll_pitch_yaw(0.0, 0.0, math.pi)}
    for k in want:
        assert np.allclose(got[k], want[k], atol=2.3e-16, rtol=0), k       # within one ulp of 0.707
        assert abs(math.sqrt(sum(v * v for v in got[k])) - 1.0) <= 1e-9          # FromDictionary's CHECK_NEAR
    # the quaternion product order: yaw * pitch * roll, not roll * pitch * yaw
    q = dliom.roll_pitch_yaw(0.3, 0.2, 0.1)
    def aa(a, axis):
        return np.array([math.cos(a / 2)] + [math.sin(a / 2) * v for v in axis])
    def mul(a, b):
        return np.array([a[0] * b[0] - a[1:] @ b[1:], *(a[0] * b[1:] + b[0] * a[1:] + np.cross(a[1:], b[1:]))])
    assert np.allclose(q, mul(mul(aa(0.1, (0, 0, 1)), aa(0.2, (0, 1, 0))), aa(0.3, (1, 0, 0))), atol=1e-15)


def decode_png(data):
    """An 8-bit RGB PNG with filter 0 -> (height, width) Cairo words, every chunk's CRC checked with zlib."""
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, chunks = 8, []
    while pos < len(data):
        n, = struct.unpack(">I", data[pos:pos + 4])
        kind, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        assert struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(kind + body)
        chunks.append((kind, body))
        pos += 12 + n
    assert [k for k, _ in chunks] == [b"IHDR", b"IDAT", b"IEND"]
    w, h, depth, ctype, comp, filt, inter = struct.unpack(">IIBBBBB", chunks[0][1])
    assert (depth, ctype, comp, filt, inter) == (8, 2, 0, 0, 0)
    raw = np.frombuffer(zlib.decompress(chunks[1][1]), np.uint8).reshape(h, 1 + 3 * w)
    assert (raw[:, 0] == 0).all()
    rgb = raw[:, 1:].reshape(h, w, 3).astype(np.uint32)
    return 0xFF000000 | rgb[..., 0] << 16 | rgb[..., 1] << 8 | rgb[..., 2]


@pytest.mark.parametrize("shape", [(1, 1), (3, 5), (70, 400)])     # 70 x 400: 84 070 bytes, two stored blocks
def test_png_round_trip(tmp_path, shape):
    import dliom
    rng = np.random.default_rng(shape[1])
    img = (0xFF000000 | rng.integers(0, 1 << 24, shape)).astype(np.uint32)
    path = tmp_path / "x.png"
    dliom.write_png(str(path), img)
    data = path.read_bytes()
    assert decode_png(data).tolist() == img.tolist()
    with pytest.raises(ValueError):
        dliom.png_bytes(np.zeros((0, 0), np.uint32))


def test_png_checksums_match_zlib():
    import dliom
    data = np.random.default_rng(5).integers(0, 256, 100_003).astype(np.uint8).tobytes()
    assert dliom._crc32(data) == zlib.crc32(data) and dliom._adler32(data) == zlib.adler32(data)


CPP_CHECK = r"""
#include <cstdio>
#include <vector>
#include "dliom_b200.hpp"
// argv: raw uint32 words file, width, height, output .png; prints RollPitchYaw of transform.lua's transforms in %a
int main(int argc, char** argv) {
  const int w = std::atoi(argv[2]), h = std::atoi(argv[3]);
  std::vector<uint32_t> argb((size_t)w * h);
  std::FILE* f = std::fopen(argv[1], "rb");
  if (!f || std::fread(argb.data(), 4, argb.size(), f) != argb.size()) return 3;
  std::fclose(f);
  const std::vector<uint8_t> png = dliom::io::PngBytes(argb, w, h);
  f = std::fopen(argv[4], "wb");
  if (!f || std::fwrite(png.data(), 1, png.size(), f) != png.size()) return 3;
  std::fclose(f);
  const double angles[3][3] = {{0., -M_PI / 2., 0.}, {0., 0., -M_PI / 2}, {0., 0., M_PI}};
  for (const auto& a : angles) {
    const std::array<double, 4> q = dliom::transform::RollPitchYaw(a[0], a[1], a[2]);
    std::printf("%a %a %a %a\n", q[0], q[1], q[2], q[3]);
  }
  return 0;
}
"""


def test_cpp_png_bytes_and_roll_pitch_yaw_match_python(tmp_path):
    import dliom
    src = tmp_path / "check.cc"
    src.write_text(CPP_CHECK)
    exe = str(tmp_path / "check")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "d-liom_b200", "host"),
                           str(src), "-o", exe, "-L" + os.path.join(ROOT, "d-liom_b200"), "-ldliom_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "d-liom_b200")])
    img = (0xFF000000 | np.random.default_rng(9).integers(0, 1 << 24, (90, 300))).astype(np.uint32)
    raw = tmp_path / "img.bin"
    raw.write_bytes(img.tobytes())
    r = subprocess.run([exe, str(raw), "300", "90", str(tmp_path / "cpp.png")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "cpp.png").read_bytes() == dliom.png_bytes(img)
    got = [tuple(float.fromhex(v) for v in line.split()) for line in r.stdout.split("\n") if line]
    want = [dliom.roll_pitch_yaw(0.0, -math.pi / 2.0, 0.0), dliom.roll_pitch_yaw(0.0, 0.0, -math.pi / 2),
            dliom.roll_pitch_yaw(0.0, 0.0, math.pi)]
    assert got == [tuple(w) for w in want]


# ---- C-ABI surface without a device
def test_xray_layouts_match_header():
    import dliom
    assert ctypes.sizeof(dliom.MapWriterColor) == 8
    assert ctypes.sizeof(dliom.MapWriterXray) == 64
    assert dliom.MapMessage.frame_id.offset == 3 * 8 + 4


def test_xray_argument_checks_without_a_writer():
    import dliom
    L = dliom.lib()
    c, x, s, w, h = dliom.MapWriterColor(), dliom.MapWriterXray(), ctypes.c_int32(0), ctypes.c_int32(0), ctypes.c_int32(0)
    assert L.dl_map_writer_add_color(None, ctypes.byref(c)) == -2
    assert L.dl_map_writer_add_xray(None, ctypes.byref(x), ctypes.byref(s)) == -2
    assert L.dl_map_writer_xray_image(None, 0, 0, None, ctypes.byref(w), ctypes.byref(h)) == -2


def test_xray_example_is_built_and_fails_loudly_without_a_gpu(tmp_path):
    import torch
    import __graft_entry__
    from test_map_writer_oracle import write_map_input
    assert os.access(__graft_entry__.XRAY_EXAMPLE, os.X_OK)
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    path = str(tmp_path / "input.bin")
    write_map_input(path, {0: ([0, 10], [IDENTITY, IDENTITY])}, [(5, 0, 1, 0, IDENTITY)], np.zeros((1, 4), np.float32))
    r = subprocess.run([__graft_entry__.XRAY_EXAMPLE, path, str(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 2 and "dliom error -1" in r.stderr
