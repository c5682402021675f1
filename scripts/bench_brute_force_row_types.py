"""Brute force over float32, float16, uint8 and int8 rows: search time, tc_scan kernel time and device bytes per row type.

    python scripts/bench_brute_force_row_types.py [--out bench_brute_force_row_types.json] [--rounds 3] [--skip-10m]

Data: bench.py's brute-force workload (gen_clustered, 1M x 128, batches of 10k queries) at k = 10 and 64, and the same generator
at 10M x 128 at k = 10.  The 8-bit rows are the fp32 rows scaled to the type's range and rounded.  Variants run in alternating
rounds; every narrow variant's ids and distances must be byte-identical to a float32 index over the same widened values.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import gen_clustered  # noqa: E402
from cuvs_b200._capi import check, lib  # noqa: E402
from cuvs_b200.neighbors import brute_force  # noqa: E402


def to_type(x, dtype, lo, hi):
    if dtype == np.float32:
        return x
    if dtype == np.float16:
        return x.astype(np.float16)
    info = np.iinfo(dtype)
    return np.clip(np.rint((x - lo) / (hi - lo) * (info.max - info.min) + info.min), info.min, info.max).astype(dtype)


def info(index):
    rt, nb = C.c_int(-1), C.c_int64(-1)
    check(lib.cuvsB200BruteForceIndexInfo(index._p, C.byref(rt), C.byref(nb)))
    return rt.value, nb.value


def timed_search(index, q, k, batch):
    lib.cuvsB200TimingTotalMs.restype = C.c_double
    lib.cuvsB200TimingReset()
    lib.cuvsB200TimingEnable(1)
    outs = []
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for b in range(0, q.shape[0], batch):
        outs.append(brute_force.search(index, q[b:b + batch], k))
    t1.record()
    torch.cuda.synchronize()
    lib.cuvsB200TimingEnable(0)
    cnt = C.c_int(0)
    scan_ms = lib.cuvsB200TimingTotalMs(b"tc_scan", C.byref(cnt))
    d = torch.cat([o[0] for o in outs]).cpu().numpy()
    i = torch.cat([o[1] for o in outs]).cpu().numpy()
    return t0.elapsed_time(t1), scan_ms, d, i


def run(n, k_list, rounds, nq, batch):
    g = torch.Generator(device="cuda")
    g.manual_seed(99)
    centers = torch.randn((max(1, n // 1000), 128), generator=g, device="cuda")  # as bench.py's BruteForceWorkload
    base = gen_clustered(n, 128, 1234, centers).cpu().numpy()
    qbase = gen_clustered(nq, 128, 1234 + 3087, centers).cpu().numpy()
    lo, hi = float(min(base.min(), qbase.min())), float(max(base.max(), qbase.max()))
    rows = []
    variants = {}
    for dt in (np.float32, np.float16, np.uint8, np.int8):
        ds, qs = to_type(base.astype(np.float32), dt, lo, hi), to_type(qbase.astype(np.float32), dt, lo, hi)
        ix = brute_force.build(torch.from_numpy(ds).cuda())
        ref = brute_force.build(torch.from_numpy(ds.astype(np.float32)).cuda()) if dt != np.float32 else None
        variants[np.dtype(dt).name] = (ix, ref, torch.from_numpy(qs).cuda(), torch.from_numpy(qs.astype(np.float32)).cuda())
    for k in k_list:
        times = {name: [] for name in variants}
        for name, (ix, ref, q, qf) in variants.items():  # warm-up, and the identity check
            _, _, d, i = timed_search(ix, q, k, batch)
            if ref is not None:
                _, _, d2, i2 = timed_search(ref, qf, k, batch)
                assert d.tobytes() == d2.tobytes() and i.tobytes() == i2.tobytes(), f"{name}: differs from float32 at k={k}"
        for _ in range(rounds):
            for name, (ix, ref, q, qf) in variants.items():
                ms, scan, _, _ = timed_search(ix, q, k, batch)
                times[name].append((ms, scan))
        for name, (ix, ref, q, qf) in variants.items():
            rt, nbytes = info(ix)
            t = times[name]
            rows.append({"n": n, "dim": 128, "k": k, "rows": name, "search_ms": [round(a, 3) for a, _ in t],
                         "tc_scan_ms": [round(b, 3) for _, b in t], "device_bytes": nbytes,
                         "bytes_per_row": round(nbytes / n, 1), "identical_to_float32": True})
            print(json.dumps(rows[-1]), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="bench_brute_force_row_types.json", help="JSON file of the results")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-10m", action="store_true")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"# {gpu}", flush=True)
    rows = run(1_000_000, (10, 64), a.rounds, 10_000, 10_000)
    if not a.skip_10m:
        rows += run(10_000_000, (10,), a.rounds, 10_000, 10_000)
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump({"gpu": gpu, "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
