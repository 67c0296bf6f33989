"""bench.py --dump-outputs: what the timed step returned, written as float32 / float64 .npy files (CPU-side check)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_dump_outputs_writes_every_returned_array(tmp_path):
    sys.path.insert(0, ROOT)
    import bench
    import dliom
    results = (dliom.ScanResult * 3)()
    results[1].pose_estimate_local[3] = 1.0
    results[1].summary.final_cost = 0.5
    results[2].num_returns = 7
    table = (dliom.ConstraintRow * 2)()
    table[1].node_id, table[1].found, table[1].score = 17, 1, 0.25
    states = np.arange(48.0).reshape(3, 16)
    bench.dump_outputs(str(tmp_path), results, states, table)
    got = {f[:-4]: np.load(os.path.join(tmp_path, f)) for f in os.listdir(tmp_path)}
    assert all(a.dtype in (np.float32, np.float64) for a in got.values())
    assert sum(a.nbytes for a in got.values()) < 64 << 20
    assert np.array_equal(got["states"], states)
    assert got["pose_estimate_local"].shape == (3, 7) and got["pose_estimate_local"][1, 3] == 1.0
    assert got["final_cost"].tolist() == [0.0, 0.5, 0.0]
    assert got["result_counts"][2, 2] == 7                     # ok, num_first_filter, num_returns, ...
    assert got["constraint_ids"][1].tolist() == [0, 17, 1, 0]  # submap_id, node_id, found, rank
    assert got["constraint_scores"][1, 0] == np.float32(0.25)
