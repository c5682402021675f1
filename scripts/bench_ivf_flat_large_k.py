#!/usr/bin/env python
"""Cost of IVF-Flat search with k > 64 (store scan into dense score segments + segmented select) at the ivf_flat bench shape.

    python scripts/bench_ivf_flat_large_k.py --out-dir DIR [--n 10000000] [--steps 5] [--rounds 3]

bench.py's ivf_flat workload: manifold data, 10M x 128, n_lists 4096, n_probes 64, batch 10k.  Searches at k in
{10, 64, 100, 256, 1024}; every shape is run once before any timing.  Per case and round: ms per batch (CUDA events), the mean
per-batch time of the `ivf_flat_scan` and `select_k_segments` sections (cuvsB200Timing*), the number of workspace batches the
search split the 10k queries into (scan sections per search), recall@k against exact ground truth on the first
`--gt-queries` queries, and for 32 < k <= 64 the share of queries the certificate sent to the store path (`flagged`).  The whole set of cases is repeated `--rounds` times.  The card's name and power limit are read in the
same run.  Output: stdout and DIR/bench_ivf_flat_large_k.json.
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


def exact_l2_ids(dataset, queries, k, chunk=2_000_000):
    """Exact squared-L2 kNN ids in fp32 (no TF32), the dataset taken in chunks and the per-chunk top-k merged."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    best_d = best_i = None
    for c0 in range(0, dataset.shape[0], chunk):
        x = dataset[c0:c0 + chunk]
        d = torch.addmm((x * x).sum(1).unsqueeze(0), queries, x.t(), beta=1.0, alpha=-2.0)
        d, i = d.topk(min(k, x.shape[0]), dim=1, largest=False)
        i = i + c0
        if best_d is None:
            best_d, best_i = d, i
        else:
            dd, ii = torch.cat([best_d, d], 1), torch.cat([best_i, i], 1)
            sel = dd.topk(k, dim=1, largest=False).indices
            best_d, best_i = dd.gather(1, sel), ii.gather(1, sel)
    torch.backends.cuda.matmul.allow_tf32 = prev
    torch.cuda.synchronize()
    return best_i


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--gt-queries", type=int, default=1000)
    ap.add_argument("--n-lists", type=int, default=4096)
    ap.add_argument("--n-probes", type=int, default=64)
    ap.add_argument("--ks", default="10,64,100,256,1024")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1234)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ivf_flat_large_k.py measures on the GPU and found none")
    os.makedirs(args.out_dir, exist_ok=True)
    ks = [int(k) for k in args.ks.split(",")]

    from cuvs_b200._capi import lib
    from cuvs_b200.common import Resources
    from cuvs_b200.neighbors import ivf_flat
    lib.cuvsB200TimingTotalMs.restype = C.c_double
    torch.cuda.set_device(0)
    dev = card(0)
    print(json.dumps({"card": dev}), flush=True)
    res = Resources()

    dataset = gen_manifold(args.n, args.d, args.seed)
    queries = gen_manifold(args.nq, args.d, args.seed + 3087)
    gt = exact_l2_ids(dataset, queries[:args.gt_queries].contiguous(), max(ks))
    torch.cuda.empty_cache()
    t0 = time.time()
    index = ivf_flat.build(ivf_flat.IndexParams(n_lists=args.n_lists, kmeans_n_iters=10,
                                                kmeans_trainset_fraction=min(0.5, max(2_000_000, 128 * args.n_lists) / args.n)),
                           dataset)
    torch.cuda.synchronize()
    print(json.dumps({"build_s": round(time.time() - t0, 1)}), flush=True)
    sp = ivf_flat.SearchParams(n_probes=args.n_probes)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    out = {k: (torch.empty((args.nq, k), dtype=torch.int64, device="cuda"), torch.empty((args.nq, k), dtype=torch.float32, device="cuda"))
           for k in ks}

    def step(k):
        ivf_flat.search(sp, index, queries, k, neighbors=out[k][0], distances=out[k][1], resources=res)

    def section(name):
        cnt = C.c_int(0)
        total = lib.cuvsB200TimingTotalMs(name, C.byref(cnt))
        return total, cnt.value

    def run(k, rnd):
        lib.cuvsB200TimingReset()
        lib.cuvsB200TimingEnable(1)
        total = 0.0
        for _ in range(args.steps):
            flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            step(k)
            res.sync()
            e.record()
            e.synchronize()
            total += s.elapsed_time(e)
        lib.cuvsB200TimingEnable(0)
        scan_ms, scans = section(b"ivf_flat_scan")
        sel_ms, _ = section(b"select_k_segments")
        found = out[k][0][:args.gt_queries]
        rec = (found.unsqueeze(2) == gt[:, :k].unsqueeze(1)).any(dim=2).float().mean().item()
        row = {"round": rnd, "k": k, "ms_per_batch": round(total / args.steps, 2), "ivf_flat_scan_ms": round(scan_ms / args.steps, 2),
               "select_k_segments_ms": round(sel_ms / args.steps, 2), "workspace_batches": scans // args.steps,
               f"recall@{k}": round(rec, 4)}
        if 32 < k <= 64:
            row["flagged"] = round(lib.cuvsB200LastFlagged() / args.nq, 4)
        print(json.dumps(row), flush=True)
        return row

    for k in ks:  # every shape once (allocator pools, kernel attributes, first-touch) before any timing
        for _ in range(args.warmup):
            step(k)
    res.sync()
    rows = [run(k, r) for r in range(args.rounds) for k in ks]
    with open(os.path.join(args.out_dir, "bench_ivf_flat_large_k.json"), "w") as f:
        json.dump({"card": dev, "args": vars(args), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
