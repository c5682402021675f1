#!/usr/bin/env python
"""Cost of IVF-PQ search with k > 64 (dense score segments + segmented select) at the flagship shape.

    python scripts/bench_ivf_pq_large_k.py --out-dir DIR [--n 50000000] [--steps 5] [--lut-dtype f16]

Flagship parameters: bench.py's manifold data, 50M x 128, n_lists 8192, pq_dim 64, n_probes 48, batch 10k.  Searches at
k in {64, 100, 256, 1024}, then search + exact refine for 100 <- 400 and 10 <- 1000 candidates.  Per case: ms per batch (CUDA
events), the mean per-batch time of the `pq_scan` and `select_k_segments` sections (cuvsB200Timing*), the number of workspace
batches the search split the 10k queries into (scan launches per search), and recall@min(k, 100) against exact ground truth on the
first `--gt-queries` queries.  The card's name and power limit are read in the same run.  Output: stdout and
DIR/bench_ivf_pq_large_k.json.
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import gen_manifold  # noqa: E402
from bench_ivf_pq_cosine import card, exact_ground_truth  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--n", type=int, default=50_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--gt-queries", type=int, default=1000)
    ap.add_argument("--n-lists", type=int, default=8192)
    ap.add_argument("--pq-dim", type=int, default=64)
    ap.add_argument("--n-probes", type=int, default=48)
    ap.add_argument("--lut-dtype", choices=["f32", "f16"], default="f16")
    ap.add_argument("--data-rank", type=int, default=16)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=1234)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ivf_pq_large_k.py measures on the GPU and found none")
    os.makedirs(args.out_dir, exist_ok=True)

    from cuvs_b200._capi import lib
    from cuvs_b200.common import Resources
    from cuvs_b200.neighbors import ivf_pq, refine
    lib.cuvsB200TimingTotalMs.restype = C.c_double
    torch.cuda.set_device(0)
    dev = card(0)
    print(json.dumps({"card": dev}), flush=True)
    res = Resources()

    dataset = gen_manifold(args.n, args.d, args.seed, rank=args.data_rank)
    queries = gen_manifold(args.nq, args.d, args.seed + 3087, rank=args.data_rank)
    gt = exact_ground_truth(dataset, queries[:args.gt_queries].contiguous(), 100, "sqeuclidean")
    torch.cuda.empty_cache()
    t0 = time.time()
    train_fraction = min(0.5, max(4_000_000, 256 * args.n_lists) / args.n)
    index = ivf_pq.build(ivf_pq.IndexParams(n_lists=args.n_lists, pq_dim=args.pq_dim, pq_bits=8, kmeans_n_iters=10,
                                            kmeans_trainset_fraction=train_fraction), dataset)
    torch.cuda.synchronize()
    print(json.dumps({"build_s": round(time.time() - t0, 1), "streamed": index.streamed}), flush=True)

    lut = {"f32": np.float32, "f16": np.float16}[args.lut_dtype]
    sp = ivf_pq.SearchParams(n_probes=args.n_probes, lut_dtype=lut)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def recall(ids, k):  # recall@min(k, 100): the first min(k, 100) columns against the exact top min(k, 100)
        k = min(k, 100)
        found = ids[:args.gt_queries, :k]
        return (found.unsqueeze(2) == gt[:, :k].unsqueeze(1)).any(dim=2).float().mean().item()

    def section(name):
        cnt = C.c_int(0)
        total = lib.cuvsB200TimingTotalMs(name, C.byref(cnt))
        return total, cnt.value

    def run(label, kc, k):
        cand = torch.empty((args.nq, kc), dtype=torch.int64, device="cuda")
        cand_d = torch.empty((args.nq, kc), dtype=torch.float32, device="cuda")
        out = torch.empty((args.nq, k), dtype=torch.int64, device="cuda")
        out_d = torch.empty((args.nq, k), dtype=torch.float32, device="cuda")

        def step():
            ivf_pq.search(sp, index, queries, kc, neighbors=cand, distances=cand_d, resources=res)
            if k != kc:
                refine(dataset, queries, cand, indices=out, distances=out_d, resources=res)

        for _ in range(args.warmup):
            step()
        res.sync()
        lib.cuvsB200TimingReset()
        lib.cuvsB200TimingEnable(1)
        total = 0.0
        for _ in range(args.steps):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            step()
            res.sync()
            e.record()
            e.synchronize()
            total += s.elapsed_time(e)
        lib.cuvsB200TimingEnable(0)
        scan_ms, scans = section(b"pq_scan")
        sel_ms, _ = section(b"select_k_segments")
        row = {"case": label, "ms_per_batch": round(total / args.steps, 2), "pq_scan_ms": round(scan_ms / args.steps, 2),
               "select_k_segments_ms": round(sel_ms / args.steps, 2), "workspace_batches": scans // args.steps,
               f"recall@{min(k, 100)}": round(recall(out if k != kc else cand, k), 4)}
        print(json.dumps(row), flush=True)
        del cand, cand_d, out, out_d
        torch.cuda.empty_cache()
        return row

    rows = [run(f"search k={k}", k, k) for k in (64, 100, 256, 1024)]
    rows += [run("search k=400 + refine to 100", 400, 100), run("search k=1000 + refine to 10", 1000, 10)]
    with open(os.path.join(args.out_dir, "bench_ivf_pq_large_k.json"), "w") as f:
        json.dump({"card": dev, "args": vars(args), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
