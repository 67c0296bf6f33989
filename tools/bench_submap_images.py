"""Submap images on the device: every submap's two textures (dl_submap_textures, Submap3D::ToResponseProto) and its high
resolution projection (dl_submap_projections, ProjectToCvMat) in one call each, for the submaps of a synthetic multi-trajectory
drive through dl_ltb at the fork's submap settings (num_range_data 100, high resolution 0.2 m, low resolution 0.45 m).

Reports, per call kind: the median and spread (min, max) of the wall-clock time of a whole call (the Python method: its size
query and its fill call, each ending in a device synchronise), after warm-up, and the grid cells per second that time covers.
Next to them: dl_grid_export_cells on the same grids, which downloads a grid's host mirror when the device is ahead (the first
export after the drive) and then walks it; that is the least any host-side rebuild of these images pays before it starts. The
GPU's name and power limit are printed with the numbers. Prints one JSON line.

    python tools/bench_submap_images.py --trajectories 4 --scans 230 --beams 16 --runs 10 --warmup 2
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "d-liom_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_ltb_batch import make_steps  # noqa: E402
from bench_map_writer import gpu_info  # noqa: E402

NOISE = [3.99e-2, 1.56e-2, 6.4e-5, 3.6e-5]


def drive(ctx, trajectories, scans, beams):
    """Builders after `scans` scans each, trajectory j starting 0.7 s after j - 1."""
    import dliom
    import imu_synth
    import orc
    import synth
    fo = dliom.FrontendOptions.from_oracle(orc.FrontEndOptions.defaults())
    opts = dliom.LtbOptions.defaults(fo, NOISE, imu_weight=0.7, num_range_data=100, high_resolution=0.2, low_resolution=0.45,
                                     max_time_seconds=0.05)
    builders = []
    for j in range(trajectories):
        b = dliom.LocalTrajectoryBuilder(ctx, opts)
        b.set_initial_state(imu_synth.state(2.0 + 0.7 * j - 0.1))
        builders.append(b)
    for row in make_steps(synth.Scene(42), trajectories, beams, scans):
        for b, (_, imu, _) in zip(builders, row):
            for t, a, g in imu:
                b.add_imu_data(t, a, g)
        dliom.add_range_data_batch(builders, [t for t, _, _ in row], [x for _, _, x in row])
    return builders


def timed(fn, runs, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trajectories", type=int, default=4)
    ap.add_argument("--scans", type=int, default=230)
    ap.add_argument("--beams", type=int, default=16)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import dliom
    ctx = dliom.Context(0)
    builders = drive(ctx, a.trajectories, a.scans, a.beams)
    submaps = [b.submap(i) for b in builders for i in range(b.num_submaps())]
    tex_queries = [(g, pose) for hi, lo, pose, _, _ in submaps for g in (hi, lo)]
    proj_queries = [(hi, pose) for hi, _, pose, _, _ in submaps]
    grids = [g for g, _ in tex_queries]
    t0 = time.perf_counter()
    cells = [len(g.export()[0]) for g in grids]   # first export after the drive: downloads every grid, then walks it
    export_cold = time.perf_counter() - t0
    export_warm = timed(lambda: [g.export() for g in grids], a.runs, a.warmup)
    tex_cells, proj_cells = sum(cells), sum(cells[0::2])
    tex = timed(lambda: ctx.submap_textures(tex_queries), a.runs, a.warmup)
    proj = timed(lambda: ctx.project_submaps(proj_queries), a.runs, a.warmup)
    before = ctx.launches
    ctx.submap_textures(tex_queries)
    launches = ctx.launches - before
    print(json.dumps({
        "gpu": gpu_info(), "trajectories": a.trajectories, "scans_per_trajectory": a.scans, "beams": a.beams,
        "submaps": len(submaps), "texture_queries": len(tex_queries), "projection_queries": len(proj_queries),
        "grid_cells_textures": tex_cells, "grid_cells_projections": proj_cells,
        "textures_call_s": {"median": tex[0], "min": tex[1], "max": tex[2]},
        "textures_cells_per_s": tex_cells / tex[0],
        "projections_call_s": {"median": proj[0], "min": proj[1], "max": proj[2]},
        "projections_cells_per_s": proj_cells / proj[0],
        "kernel_launches_per_texture_call": launches,
        "export_cells_first_s": export_cold,
        "export_cells_s": {"median": export_warm[0], "min": export_warm[1], "max": export_warm[2]},
    }))
    for b in builders:
        b.close()


if __name__ == "__main__":
    main()
