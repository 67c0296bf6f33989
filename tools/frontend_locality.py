"""How local are the front end's voxel duplicates in input order? (CPU only, numpy.)

For one bench scan (synth.make_scan(synth.Scene(42), 64, 2.05): azimuth-major firing order) and both voxel filters of the front
half (first: voxel_filter_size / 2 on the raw rows; second: voxel_filter_size, with the raw frame standing in for the deskewed
one), prints the survivors, the share of duplicates whose winner (lowest index of the voxel) lies in the duplicate's own tile,
and the scan-wide inserts left after a per-tile de-duplication (one per distinct voxel per tile). np.round (ties to even) stands
in for lroundf, so the counts are approximate.

    python tools/frontend_locality.py [--tiles 1024 2048 4096]
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def first_per_voxel(xyz, res):
    cells = np.round(xyz / np.float32(res)).astype(np.int64)
    _, inverse = np.unique(cells, axis=0, return_inverse=True)
    inverse = inverse.reshape(-1)
    winner = np.full(inverse.max() + 1, len(xyz), np.int64)
    np.minimum.at(winner, inverse, np.arange(len(xyz)))
    return inverse, winner


def locality(xyz, rows, res, tile):
    """rows: the input row of every point (the tiles are tiles of input rows, as in the kernels)."""
    inverse, winner = first_per_voxel(xyz, res)
    dup = winner[inverse] != np.arange(len(xyz))
    same_tile = (rows[winner[inverse]] // tile) == (rows // tile)
    tile_inserts = len(np.unique(inverse * (rows[-1] // tile + 1) + rows // tile))
    return len(winner), int(dup.sum()), int((dup & same_tile).sum()), tile_inserts


def main():
    import synth
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, nargs="+", default=[1024, 2048, 4096])
    ap.add_argument("--voxel", type=float, default=0.15)
    args = ap.parse_args()
    rows = synth.make_scan(synth.Scene(42), 64, 2.05)
    xyz = np.stack([rows["x"], rows["y"], rows["z"]], 1).astype(np.float32)
    n = len(xyz)
    _, first_winner = first_per_voxel(xyz, args.voxel / 2)
    kept_rows = np.sort(first_winner)
    print(f"rows {n}")
    for name, pts, rows_of, res in (("first filter", xyz, np.arange(n), args.voxel / 2),
                                    ("second filter", xyz[kept_rows], kept_rows, args.voxel)):
        for tile in args.tiles:
            kept, dups, local, inserts = locality(pts, rows_of, res, tile)
            print(f"{name:13s} res {res:.3f} m  tile {tile:5d}: survivors {kept} of {len(pts)} ({100 * kept / len(pts):.1f} %), "
                  f"duplicates with the winner in their tile {100 * local / max(dups, 1):.1f} %, "
                  f"scan-wide inserts {inserts} instead of {len(pts)} ({100 * (inserts - len(pts)) / len(pts):+.0f} %)")


if __name__ == "__main__":
    main()
