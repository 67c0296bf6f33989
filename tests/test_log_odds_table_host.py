"""The texture kernel's ProbabilityToLogOddsInteger is a host-built table of float thresholds (d-liom_b200/csrc/dl_log_odds.h):
checked here on the CPU against the reference's expression with glibc logf for every float of [kMinProbability,
kMaxProbability]. The device lookup is the same inline function, checked end to end in tests/test_gpu_submap_images.py."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_log_odds_table_equals_the_reference_for_every_float(tmp_path):
    exe = str(tmp_path / "log_odds_table_check")
    # the reference's flags: no -march, no fast-math, no contraction (cmake/functions.cmake:75,92-95)
    subprocess.check_call(["g++", "-O3", "-std=c++17", "-ffp-contract=off", "-x", "c++",
                           os.path.join(ROOT, "tests", "cpp", "log_odds_table_check.cc"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "bad=0" in out.stdout
    assert "steps=255" in out.stdout
