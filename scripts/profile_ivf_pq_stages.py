"""Stage timeline of one bench.py search step: where the device time of a batch goes, and how long the stream sits idle.

    python scripts/profile_ivf_pq_stages.py [--workload ivf_pq|ivf_pq_c2|ivf_flat] [--steps 5] [--warmup 5] [--trace FILE]

The workload is bench.py's own (same generators, seeds and parameters; the default is the flagship IVF-PQ 50M x 128 search
followed by the exact refine).  After a warm-up, each step is run once under torch.profiler with CUDA activities, with the
same 256 MiB L2 flush in front of it as in bench.py, and the GPU activities of the step (kernels, memsets, copies) give:
  - every kernel's device time per step (mean over the profiled steps) and launches per step;
  - the sum of activity time, and the idle time of the stream between the step's first and last activity;
and, in a separate loop without the profiler, the step's time between CUDA events (as bench.py takes it).  The card's name
and power limit are read in the same run: a time means little without them.
"""
import argparse
import os
import re
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench  # noqa: E402


def card():
    idx = torch.cuda.current_device()
    out = subprocess.run(["nvidia-smi", f"--id={idx}", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return out or torch.cuda.get_device_name(idx)


def short_name(name):
    """`void ns::(anonymous namespace)::kern<...>(args)` -> `kern`"""
    name = re.sub(r"^void ", "", name)
    depth, out = 0, []
    for ch in name:  # drop template arguments and the parameter list
        if ch in "<(":
            depth += 1
        elif ch in ">)":
            depth -= 1
        elif depth == 0:
            out.append(ch)
    base = "".join(out).split("::")[-1].strip()
    return base or name


def gpu_activities(prof):
    """(name, start_ns, end_ns) of every device-side activity the profiler saw, in start order."""
    acts = []
    for e in prof.profiler.kineto_results.events():
        if e.device_type() != torch.autograd.DeviceType.CUDA or e.duration_ns() <= 0:
            continue
        acts.append((short_name(e.name()), e.start_ns(), e.end_ns()))
    acts.sort(key=lambda a: a[1])
    return acts


def busy_ns(acts):
    """union of the activities' intervals (activities of other streams would overlap; the search uses one)"""
    total, cur_s, cur_e = 0, None, None
    for _, s, e in acts:
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                total += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    if cur_e is not None:
        total += cur_e - cur_s
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="ivf_pq", choices=["ivf_pq", "ivf_pq_c2", "ivf_flat"])
    ap.add_argument("--steps", type=int, default=5, help="profiled steps, and CUDA-event timed steps (x 4)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--trace", default="", help="also write the last profiled step's chrome trace here")
    args = ap.parse_args()

    from cuvs_b200.common import Resources
    torch.cuda.set_device(0)
    res = Resources()
    wl = bench.WORKLOADS[args.workload](resources=res)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    print(f"card: {card()}")
    print(f"workload: {wl.name}")
    for _ in range(args.warmup):
        wl.step(res)
    res.sync()

    # step time between CUDA events, profiler off (bench.py's timed loop)
    ev_ms = []
    for _ in range(4 * args.steps):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        wl.step(res)
        res.sync()
        e.record()
        e.synchronize()
        ev_ms.append(s.elapsed_time(e))

    per_kernel = defaultdict(lambda: [0.0, 0])  # name -> [total ns, launches]
    order = {}
    spans, busies = [], []
    for i in range(args.steps):
        flush.zero_()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            wl.step(res)
            res.sync()
        acts = gpu_activities(prof)
        if not acts:
            raise SystemExit("the profiler saw no GPU activity: CUPTI unavailable?")
        for name, s, e in acts:
            order.setdefault(name, len(order))
            per_kernel[name][0] += e - s
            per_kernel[name][1] += 1
        spans.append(acts[-1][2] - acts[0][1])
        busies.append(busy_ns(acts))
        if args.trace and i == args.steps - 1:
            prof.export_chrome_trace(args.trace)

    n = args.steps
    print(f"\nper step, mean of {n} profiled steps (device time of each activity, in first-launch order):")
    print(f"{'activity':<40} {'launches':>8} {'ms':>9}")
    for name in sorted(per_kernel, key=lambda k: order[k]):
        t, c = per_kernel[name]
        print(f"{name[:40]:<40} {c / n:>8.1f} {t / n / 1e6:>9.4f}")
    span, busy = sum(spans) / n / 1e6, sum(busies) / n / 1e6
    print(f"{'sum of activity time':<49} {sum(v[0] for v in per_kernel.values()) / n / 1e6:>9.4f}")
    print(f"{'busy (union of activities)':<49} {busy:>9.4f}")
    print(f"{'idle between first and last activity':<49} {span - busy:>9.4f}")
    print(f"{'first activity start to last activity end':<49} {span:>9.4f}")
    ev_ms.sort()
    print(f"{'step, CUDA events (profiler off), median':<49} {ev_ms[len(ev_ms) // 2]:>9.4f}"
          f"   (min {ev_ms[0]:.4f}, max {ev_ms[-1]:.4f}, {len(ev_ms)} steps)")


if __name__ == "__main__":
    main()
