#!/usr/bin/env python
"""IVF-Flat on uint8 rows stored as bytes and scanned on the integer tensor cores, against a float32 index of the same values.

    python scripts/bench_ivf_flat_u8.py --out-dir DIR [--n 10000000] [--rounds 3] [--big 100000000]

The ivf_flat bench shape: 10M x 128, n_lists 4096, n_probes 64, batch 10k, k 10 and 100.  The rows are bench.py's manifold
data mapped to uint8 (x * 40 + 128, rounded and clamped), generated on the device.  The uint8 index is built first; the float32
index gets its centres (set_centers) and the same values widened, so both probe the same lists.  Per round and k, both
indexes in turn: ms per batch (CUDA events) and the mean per-batch time of the `ivf_flat_scan` section (cuvsB200Timing*).
Once: the device bytes of each index (mem_get_info delta of a second build, after a warm-up build has filled the memory pool),
and whether the two indexes' outputs are byte-identical, or else that every difference lies in a tie group at the k-th slot.
With --big N: an N x 128 uint8 index built by extends of at most 10M rows, its build time, device bytes, and recall@10 on the
first 1000 queries against exact ground truth computed chunk-wise.  The card's name and power limit are read in the same run.
Output: stdout and DIR/bench_ivf_flat_u8.json.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from bench import gen_manifold  # noqa: E402
from bench_ivf_pq_cosine import card  # noqa: E402

CHUNK = 10_000_000


def gen_u8(n, d, seed):
    out = torch.empty((n, d), dtype=torch.uint8, device="cuda")
    for i, s in enumerate(range(0, n, CHUNK)):
        e = min(n, s + CHUNK)
        out[s:e] = (gen_manifold(e - s, d, seed + 7919 * i) * 40.0 + 128.0).round_().clamp_(0, 255).to(torch.uint8)
    return out


def exact_l2_ids(rows_u8, queries, k):
    """Exact squared-L2 kNN ids: int64-exact fp32 products (values < 2^24 at d = 128), chunk by chunk, per-chunk top-k merged."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    best_d = best_i = None
    for c0 in range(0, rows_u8.shape[0], 2_000_000):
        x = rows_u8[c0:c0 + 2_000_000].float()
        d = torch.addmm((x * x).sum(1).unsqueeze(0), queries, x.t(), beta=1.0, alpha=-2.0)
        d, i = d.topk(min(k, x.shape[0]), dim=1, largest=False)
        if best_d is None:
            best_d, best_i = d, i + c0
        else:
            dd, ii = torch.cat([best_d, d], 1), torch.cat([best_i, i + c0], 1)
            sel = dd.topk(k, dim=1, largest=False).indices
            best_d, best_i = dd.gather(1, sel), ii.gather(1, sel)
    torch.backends.cuda.matmul.allow_tf32 = prev
    return best_i


def tie_report(d8, i8, d32, i32):
    """Byte-identical, or every differing id sits in the group of distances equal to the k-th."""
    if torch.equal(d8, d32) and torch.equal(i8, i32):
        return {"identical": True}
    same_dist = torch.equal(d8.view(torch.int32), d32.view(torch.int32))
    kth = d32[:, -1:]
    differ = i8 != i32
    outside = differ & (d32 != kth)
    # inside the k-th group the members may differ; the ids before it must be the same set
    return {"identical": False, "distances_identical": bool(same_dist), "queries_with_other_ids": int(differ.any(1).sum()),
            "differences_outside_the_kth_tie_group": int(outside.sum())}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--n-lists", type=int, default=4096)
    ap.add_argument("--n-probes", type=int, default=64)
    ap.add_argument("--ks", default="10,100")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--big", type=int, default=0)
    ap.add_argument("--seed", type=int, default=1234)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ivf_flat_u8.py measures on the GPU and found none")
    os.makedirs(args.out_dir, exist_ok=True)
    ks = [int(k) for k in args.ks.split(",")]

    from cuvs_b200._capi import lib
    from cuvs_b200.common import Resources
    from cuvs_b200.neighbors import ivf_flat
    lib.cuvsB200TimingTotalMs.restype = C.c_double
    torch.cuda.set_device(0)
    dev = card(0)
    report = {"card": dev, "args": vars(args)}
    print(json.dumps({"card": dev}), flush=True)
    res = Resources()

    rows8 = gen_u8(args.n, args.d, args.seed)
    queries8 = gen_u8(args.nq, args.d, args.seed + 3087)
    queries32 = queries8.float()
    frac = min(0.5, max(2_000_000, 128 * args.n_lists) / args.n)
    params8 = ivf_flat.IndexParams(n_lists=args.n_lists, kmeans_n_iters=10, kmeans_trainset_fraction=frac)

    def measured(make):
        """(index, device bytes): the second of two builds, so that the pool already holds the build's temporaries."""
        warm = make()
        del warm
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0, _ = torch.cuda.mem_get_info()
        t0 = time.time()
        index = make()
        torch.cuda.synchronize()
        secs = time.time() - t0
        free1, _ = torch.cuda.mem_get_info()
        return index, free0 - free1, secs

    idx8, bytes8, s8 = measured(lambda: ivf_flat.build(params8, rows8))
    centers = idx8.centers.clone()
    rows32 = rows8.float()

    def make32():
        ix = ivf_flat.build(ivf_flat.IndexParams(n_lists=args.n_lists, add_data_on_build=False), rows32[:args.n_lists])
        ivf_flat.set_centers(ix, centers)
        return ivf_flat.extend(ix, rows32, None)

    idx32, bytes32, s32 = measured(make32)
    del rows32
    torch.cuda.empty_cache()
    report["index_bytes"] = {"uint8": bytes8, "float32": bytes32, "rows": args.n}
    report["build_s"] = {"uint8": round(s8, 1), "float32_extend_with_given_centres": round(s32, 1)}
    print(json.dumps({"index_bytes": report["index_bytes"], "build_s": report["build_s"]}), flush=True)

    sp = ivf_flat.SearchParams(n_probes=args.n_probes)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    out = {(t, k): (torch.empty((args.nq, k), dtype=torch.int64, device="cuda"), torch.empty((args.nq, k), dtype=torch.float32, device="cuda"))
           for t in ("uint8", "float32") for k in ks}
    cases = {"uint8": (idx8, queries8), "float32": (idx32, queries32)}

    def step(t, k):
        index, q = cases[t]
        ivf_flat.search(sp, index, q, k, neighbors=out[(t, k)][0], distances=out[(t, k)][1], resources=res)

    def run(t, k, rnd):
        lib.cuvsB200TimingReset()
        lib.cuvsB200TimingEnable(1)
        total = 0.0
        for _ in range(args.steps):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            step(t, k)
            res.sync()
            e.record()
            e.synchronize()
            total += s.elapsed_time(e)
        lib.cuvsB200TimingEnable(0)
        cnt = C.c_int(0)
        scan = lib.cuvsB200TimingTotalMs(b"ivf_flat_scan", C.byref(cnt))
        row = {"round": rnd, "index": t, "k": k, "ms_per_batch": round(total / args.steps, 2),
               "ivf_flat_scan_ms": round(scan / args.steps, 2)}
        print(json.dumps(row), flush=True)
        return row

    for t in cases:
        for k in ks:
            step(t, k)
    res.sync()
    report["rows"] = [run(t, k, r) for r in range(args.rounds) for k in ks for t in cases]
    report["outputs"] = {}
    for k in ks:
        d8, i8 = out[("uint8", k)][1], out[("uint8", k)][0]
        d32, i32 = out[("float32", k)][1], out[("float32", k)][0]
        report["outputs"][k] = tie_report(d8, i8, d32, i32)
    print(json.dumps({"outputs": report["outputs"]}), flush=True)
    del idx32, cases
    torch.cuda.empty_cache()

    if args.big:
        del idx8
        del rows8
        torch.cuda.empty_cache()
        big = gen_u8(args.big, args.d, args.seed + 17)
        free0, _ = torch.cuda.mem_get_info()
        t0 = time.time()
        first = min(CHUNK, args.big)
        index = ivf_flat.build(ivf_flat.IndexParams(n_lists=args.n_lists, kmeans_n_iters=10, add_data_on_build=False,
                                                    kmeans_trainset_fraction=min(0.5, max(2_000_000, 128 * args.n_lists) / first)),
                               big[:first])
        for s in range(0, args.big, CHUNK):
            ivf_flat.extend(index, big[s:s + CHUNK], None)
        torch.cuda.synchronize()
        build_s = time.time() - t0
        free1, _ = torch.cuda.mem_get_info()
        q = queries8[:1000].contiguous()
        _, found = ivf_flat.search(sp, index, q, 10, resources=res)
        res.sync()
        gt = exact_l2_ids(big, q.float(), 10)
        rec = (found.unsqueeze(2) == gt.unsqueeze(1)).any(dim=2).float().mean().item()
        report["big"] = {"rows": args.big, "build_s": round(build_s, 1), "index_bytes_upper_bound": free0 - free1,
                         "recall@10": round(rec, 4), "total_device_bytes": torch.cuda.mem_get_info()[1]}
        print(json.dumps({"big": report["big"]}), flush=True)

    with open(os.path.join(args.out_dir, "bench_ivf_flat_u8.json"), "w") as f:
        json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
