#!/usr/bin/env python
"""Inner product against cosine IVF-PQ on the same data, at the flagship shape.

    python scripts/bench_ivf_pq_cosine.py --out-dir DIR [--n 50000000] [--rounds 3] [--steps 20] [--lut-dtype f16]

Rows are bench.py's embedding-like manifold data times a seeded log-uniform factor in [0.1, 10] (`--norm-spread 10`), so
that the inner-product and cosine rankings really differ.  Both indexes use the flagship parameters (n_lists 8192, pq_dim 64,
n_probes 48, batch 10k, k 10, an exact refine of k x 2 candidates with the index's own metric).  Ground truth is exact brute
force with each
index's metric, run over 10M-row chunks and merged (a brute-force index over all 50M rows does not fit next to the data).
The two indexes are searched alternately, `--rounds` times each.  Per index and round the script prints the search time
(CUDA events, IVF-PQ search alone, then search + refine), the queries per second of search + refine, the `pq_scan` kernel
time (cuvsB200Timing*), recall@10 after the refine, and the build time, and per index how many list rows the coarse probes
send each query to and how unevenly the probes spread over the lists.  The card's name and power limit are read in the
same run.  Everything goes to stdout and to DIR/bench_ivf_pq_cosine.json.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import gen_manifold  # noqa: E402


def mixed_norm_rows(n, d, seed, data_rank, spread):
    x = gen_manifold(n, d, seed, rank=data_rank)
    if spread == 1.0:
        return x
    g = torch.Generator(device="cuda")
    g.manual_seed(seed + 17)
    step = 1 << 22
    for s in range(0, n, step):
        e = min(n, s + step)
        f = torch.empty(e - s, device="cuda").uniform_(-math.log(spread), math.log(spread), generator=g).exp_()
        x[s:e] *= f[:, None]
    return x


def exact_ground_truth(dataset, queries, k, metric, chunk=10_000_000):
    """Exact kNN ids by brute force with `metric`, the dataset taken in chunks and the per-chunk results merged."""
    from cuvs_b200.neighbors import brute_force
    largest = metric == "inner_product"  # brute force returns the dot product itself for inner product
    best_d = best_i = None
    for c0 in range(0, dataset.shape[0], chunk):
        bf = brute_force.build(dataset[c0:c0 + chunk], metric=metric)
        d, i = brute_force.search(bf, queries, k)
        i = i.to(torch.int64) + c0
        del bf
        if best_d is None:
            best_d, best_i = d, i
        else:
            dd, ii = torch.cat([best_d, d], 1), torch.cat([best_i, i], 1)
            sel = dd.topk(k, dim=1, largest=largest).indices
            best_d, best_i = dd.gather(1, sel), ii.gather(1, sel)
    torch.cuda.synchronize()
    return best_i


def probe_load(index, queries, n_probes):
    """Coarse probes of both metrics rank lists by -q.c: -> (list rows scanned per query, max / mean probing queries per list)."""
    c = index.centers
    sizes = index.list_sizes.to(torch.int64)
    rows, hist = 0, torch.zeros(c.shape[0], dtype=torch.int64, device=c.device)
    for s in range(0, queries.shape[0], 1000):
        p = (queries[s:s + 1000] @ c.T).topk(n_probes, dim=1).indices
        rows += sizes[p].sum().item()
        hist += torch.bincount(p.flatten(), minlength=c.shape[0])
    return rows / queries.shape[0], hist.max().item() / hist.float().mean().item()


def card(device):
    """(name, power limit, max SM clock) of the card, read with nvidia-smi; the name from torch if nvidia-smi is unavailable."""
    try:
        out = subprocess.run(["nvidia-smi", f"--id={device}", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [s.strip() for s in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(device), "power_limit": f"unknown ({type(e).__name__})", "max_sm_clock": "unknown"}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--n", type=int, default=50_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--n-lists", type=int, default=8192)
    ap.add_argument("--pq-dim", type=int, default=64)
    ap.add_argument("--n-probes", type=int, default=48)
    ap.add_argument("--refine-ratio", type=int, default=2)
    ap.add_argument("--lut-dtype", choices=["f32", "f16", "u8"], default="f16")
    ap.add_argument("--data-rank", type=int, default=16)
    ap.add_argument("--norm-spread", type=float, default=10.0, help="row norms scaled by a log-uniform factor in [1/S, S]")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1234)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ivf_pq_cosine.py measures on the GPU and found none")
    os.makedirs(args.out_dir, exist_ok=True)

    from cuvs_b200._capi import lib
    from cuvs_b200.common import Resources
    from cuvs_b200.neighbors import ivf_pq, refine
    lib.cuvsB200TimingTotalMs.restype = C.c_double
    torch.cuda.set_device(0)
    dev = card(0)
    print(json.dumps({"card": dev}), flush=True)

    res = Resources()
    n, k, kc = args.n, args.k, args.k * args.refine_ratio
    t0 = time.time()
    dataset = mixed_norm_rows(n, args.d, args.seed, args.data_rank, args.norm_spread)
    queries = mixed_norm_rows(args.nq, args.d, args.seed + 3087, args.data_rank, args.norm_spread)
    torch.cuda.synchronize()
    gen_s = time.time() - t0
    metrics = ("inner_product", "cosine")
    gt, gt_s = {}, {}
    for m in metrics:
        t0 = time.time()
        gt[m] = exact_ground_truth(dataset, queries, k, m)
        gt_s[m] = time.time() - t0
        torch.cuda.empty_cache()
    # the two rankings really differ on this data
    gt_overlap = (gt["cosine"].unsqueeze(2) == gt["inner_product"].unsqueeze(1)).any(dim=2).float().mean().item()

    train_fraction = min(0.5, max(4_000_000, 256 * args.n_lists) / n)
    index, build_s, load = {}, {}, {}
    for m in metrics:
        t0 = time.time()
        index[m] = ivf_pq.build(ivf_pq.IndexParams(n_lists=args.n_lists, pq_dim=args.pq_dim, pq_bits=8, kmeans_n_iters=10,
                                                   kmeans_trainset_fraction=train_fraction, metric=m), dataset)
        torch.cuda.synchronize()
        build_s[m] = time.time() - t0
        path, nbytes = index[m]._info()
        rows, skew = probe_load(index[m], queries, args.n_probes)
        load[m] = {"probed_rows_per_query": round(rows), "probing_queries_per_list_max_over_mean": round(skew, 2)}
        print(json.dumps({"index": m, "build_s": round(build_s[m], 2), "path": path, "device_bytes": nbytes, **load[m]}), flush=True)

    lut = {"f32": np.float32, "f16": np.float16, "u8": np.uint8}[args.lut_dtype]
    sp = ivf_pq.SearchParams(n_probes=args.n_probes, lut_dtype=lut)
    cand = torch.empty((args.nq, kc), dtype=torch.int64, device="cuda")
    cand_d = torch.empty((args.nq, kc), dtype=torch.float32, device="cuda")
    nb = torch.empty((args.nq, k), dtype=torch.int64, device="cuda")
    nd = torch.empty((args.nq, k), dtype=torch.float32, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def search(m):
        ivf_pq.search(sp, index[m], queries, kc, neighbors=cand, distances=cand_d, resources=res)

    def search_refine(m):
        search(m)
        refine(dataset, queries, cand, indices=nb, distances=nd, metric=m, resources=res)

    def timed(fn, m):
        total = 0.0
        for _ in range(args.steps):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn(m)
            res.sync()
            e.record()
            e.synchronize()
            total += s.elapsed_time(e)
        return total / args.steps

    runs = []
    for r in range(args.rounds):
        for m in metrics:
            for _ in range(args.warmup):
                search_refine(m)
            res.sync()
            lib.cuvsB200TimingReset()
            lib.cuvsB200TimingEnable(1)
            search_ms = timed(search, m)
            lib.cuvsB200TimingEnable(0)
            cnt = C.c_int(0)
            scan_ms = lib.cuvsB200TimingTotalMs(b"pq_scan", C.byref(cnt)) / max(cnt.value, 1)
            step_ms = timed(search_refine, m)
            recall = (nb.unsqueeze(2) == gt[m].unsqueeze(1)).any(dim=2).float().mean().item()
            row = {"round": r, "index": m, "search_ms": round(search_ms, 3), "search_refine_ms": round(step_ms, 3),
                   "qps": round(args.nq / (step_ms * 1e-3)), "pq_scan_ms": round(scan_ms, 3), "recall@10": round(recall, 4),
                   "build_s": round(build_s[m], 2)}
            runs.append(row)
            print(json.dumps(row), flush=True)

    summary = {}
    for m in metrics:
        rows = [x for x in runs if x["index"] == m]
        summary[m] = {key: [min(x[key] for x in rows), float(np.median([x[key] for x in rows])), max(x[key] for x in rows)]
                      for key in ("search_ms", "search_refine_ms", "qps", "pq_scan_ms", "recall@10")}
        summary[m]["build_s"] = round(build_s[m], 2)
        summary[m].update(load[m])
    out = {"card": dev, "config": {key: getattr(args, key) for key in ("n", "d", "nq", "k", "n_lists", "pq_dim", "n_probes",
                                                                     "refine_ratio", "lut_dtype", "data_rank", "norm_spread", "rounds", "steps",
                                                                     "warmup", "seed")},
           "data_gen_s": round(gen_s, 2), "ground_truth_s": {m: round(v, 2) for m, v in gt_s.items()},
           "ground_truth_overlap_cosine_vs_ip": round(gt_overlap, 4), "runs": runs, "summary_min_median_max": summary}
    with open(os.path.join(args.out_dir, "bench_ivf_pq_cosine.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({"summary_min_median_max": summary, "ground_truth_overlap_cosine_vs_ip": round(gt_overlap, 4)}), flush=True)


if __name__ == "__main__":
    main()
