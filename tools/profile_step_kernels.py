"""Per-kernel device time of the bench workload, from torch.profiler (CUDA activities).

Runs bench.py in this process with the given arguments (default: a short run of the headline step without the exchange and
without the extra measurements) under the profiler, and writes the kernels sorted by total device time, with calls and time per
call, to OUT. Profile in a run of its own: tracing slows the host, so take step times from bench.py without the profiler.

    python tools/profile_step_kernels.py /tmp/profile/kernels.txt [-- bench args]
"""
import os
import runpy
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    if len(sys.argv) < 2:
        sys.exit(__doc__)
    out = sys.argv[1]
    rest = sys.argv[2:]
    if rest and rest[0] == "--":
        rest = rest[1:]
    bench_args = rest or ["--steps", "20", "--warmup", "3", "--pairs", "0", "--no-extras", "--cpu-sample", "8"]
    import torch
    from torch.profiler import ProfilerActivity, profile
    sys.argv = [os.path.join(ROOT, "bench.py")] + bench_args
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        runpy.run_path(sys.argv[0], run_name="__main__")
    torch.cuda.synchronize()
    rows = []
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if t > 0:
            rows.append((t, e.count, e.key))
    rows.sort(reverse=True)
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, "w") as f:
        f.write(f"bench args: {' '.join(bench_args)}\n{'total us':>12} {'calls':>7} {'us/call':>10}  kernel\n")
        for t, n, k in rows:
            f.write(f"{t:12.1f} {n:7d} {t / n:10.2f}  {k[:110]}\n")
    print(open(out).read())


if __name__ == "__main__":
    main()
