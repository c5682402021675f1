#!/usr/bin/env python
"""NN-descent, and CAGRA built with it against the default kNN stage, at the C3 shape.

    python scripts/bench_nn_descent.py --out-dir DIR [--n 10000000] [--d 96] [--degree 64] [--dtype float32] [--dump-outputs]

Rows are bench.py's embedding-like manifold data (10M x 96), queries the same generator with another seed.  First an
NN-descent graph (graph degree --degree, intermediate 2 x degree, 20 iterations, as the reference's defaults) is built;
the script prints its total time (host clock around the call, which ends in a device synchronise), the time of each phase
from the library's CUDA-event sections (cuvsB200Timing*: init, sample, reverse, join, merge, re-score; the sample section's
count is the number of iterations run), the peak of the device's default memory pool during the build (the library's
stream-ordered temporaries, which torch's allocator statistics do not see) and the graph's recall against the exact
neighbours of 1000 sampled rows.  --dtype builds over the rows cast to float16, or scaled to the 8-bit type's range and
rounded (uint8 offset by 128); the recall is then taken against the exact neighbours of those rows.  --dump-outputs also
builds with distances and writes the graph and distances to DIR/nn_descent_graph.npy and DIR/nn_descent_distances.npy, for
comparing two builds bit for bit.  Then, for float32 rows only, a CAGRA index is built twice, build_algo "nn_descent" and the default path, both searched with itopk 64, batch 10k, k 10,
and recall@10 is taken on the first 1000 queries against exact ground truth.  Once, the card's name and power limit, read
in the same run.  Everything goes to stdout and to DIR/bench_nn_descent.json.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import gen_manifold  # noqa: E402
from bench_cagra_row_types import to_8bit  # noqa: E402
from bench_ivf_pq_cosine import card, exact_ground_truth  # noqa: E402

CU_MEMPOOL_ATTR_USED_MEM_HIGH = 8  # cudaMemPoolAttrUsedMemHigh


class PoolPeak:
    """Peak bytes in use of a device's default memory pool (where the library's cudaMallocAsync temporaries live), through the
    driver API: reset() zeroes the high-water mark, read() returns it."""

    def __init__(self, device=0):
        self.cu = C.CDLL("libcuda.so.1")
        dev, self.pool = C.c_int(0), C.c_void_p(0)
        assert self.cu.cuDeviceGet(C.byref(dev), device) == 0
        assert self.cu.cuDeviceGetDefaultMemPool(C.byref(self.pool), dev) == 0

    def reset(self):
        zero = C.c_uint64(0)
        assert self.cu.cuMemPoolSetAttribute(self.pool, CU_MEMPOOL_ATTR_USED_MEM_HIGH, C.byref(zero)) == 0

    def read(self):
        v = C.c_uint64(0)
        assert self.cu.cuMemPoolGetAttribute(self.pool, CU_MEMPOOL_ATTR_USED_MEM_HIGH, C.byref(v)) == 0
        return v.value


SECTIONS = ("nn_descent_init", "nn_descent_sample", "nn_descent_reverse", "nn_descent_join", "nn_descent_merge", "nn_descent_rescore")


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=96)
    ap.add_argument("--degree", type=int, default=64)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--gt-queries", type=int, default=1000)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--dtype", choices=("float32", "float16", "int8", "uint8"), default="float32")
    ap.add_argument("--dump-outputs", action="store_true")
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)
    from cuvs_b200._capi import lib
    from cuvs_b200.neighbors import cagra, nn_descent
    lib.cuvsB200TimingTotalMs.restype = C.c_double
    k = 10
    info = {"card": card(0), "n": args.n, "d": args.d, "degree": args.degree, "dtype": args.dtype}
    print(json.dumps(info), flush=True)
    dataset = gen_manifold(args.n, args.d, args.seed)
    queries = gen_manifold(args.nq, args.d, args.seed + 3087)
    if args.dtype == "float16":
        dataset = dataset.half()
    elif args.dtype != "float32":
        dataset = to_8bit(dataset, 127.0 / dataset.abs().max().item(), getattr(torch, args.dtype))
    peak = PoolPeak(0)

    # ---- NN-descent on its own
    torch.cuda.synchronize()
    lib.cuvsB200TimingReset()
    lib.cuvsB200TimingEnable(1)
    peak.reset()
    t0 = time.perf_counter()
    nnd = nn_descent.build(nn_descent.IndexParams(graph_degree=args.degree, intermediate_graph_degree=2 * args.degree,
                                                  return_distances=args.dump_outputs), dataset)
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
    lib.cuvsB200TimingEnable(0)
    row = {"nn_descent_build_s": round(total, 3), "pool_peak_bytes": peak.read()}
    for name in SECTIONS:
        cnt = C.c_int(0)
        row[name + "_ms"] = round(lib.cuvsB200TimingTotalMs(name.encode(), C.byref(cnt)), 2)
        if name == "nn_descent_sample":
            row["iterations"] = cnt.value
    rows = torch.from_numpy(np.random.default_rng(7).choice(args.n, args.gt_queries, replace=False)).cuda()
    rows32 = dataset.float()
    gt = exact_ground_truth(rows32, rows32[rows], args.degree + 1, "sqeuclidean").cpu().numpy()
    del rows32
    got = nnd.graph.to(torch.int64)[rows].cpu().numpy()
    hits = [len(set(g.tolist()) & set([v for v in t if v != r][:args.degree])) for g, t, r in zip(got, gt, rows.cpu().numpy())]
    row["graph_recall"] = round(float(np.sum(hits)) / (args.gt_queries * args.degree), 4)
    print(json.dumps(row), flush=True)
    info["nn_descent"] = row
    if args.dump_outputs:
        np.save(os.path.join(args.out_dir, "nn_descent_graph.npy"), nnd.graph.to(torch.int64).cpu().numpy())
        np.save(os.path.join(args.out_dir, "nn_descent_distances.npy"), nnd.distances.cpu().numpy())
    del nnd
    torch.cuda.empty_cache()
    if args.dtype != "float32":
        with open(os.path.join(args.out_dir, "bench_nn_descent.json"), "w") as f:
            json.dump(info, f, indent=1)
        return

    # ---- CAGRA: NN_DESCENT against the default kNN stage, same run
    gtq = exact_ground_truth(dataset, queries[:args.gt_queries], k, "sqeuclidean").cpu().numpy()
    sp = cagra.SearchParams(itopk_size=64)
    info["cagra"] = []
    for algo in ("nn_descent", "ivf_pq"):
        params = cagra.IndexParams(graph_degree=args.degree, intermediate_graph_degree=2 * args.degree, build_algo=algo)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        index = cagra.build(params, dataset)
        torch.cuda.synchronize()
        build_s = time.perf_counter() - t0
        _, nb = cagra.search(sp, index, queries, k)
        got = nb[:args.gt_queries].to(torch.int64).cpu().numpy()
        rec = float(np.mean([len(set(a) & set(b)) / k for a, b in zip(got, gtq)]))
        r = {"build_algo": algo if algo == "nn_descent" else "default", "cagra_build_s": round(build_s, 3), "recall@10": round(rec, 4)}
        print(json.dumps(r), flush=True)
        info["cagra"].append(r)
        del index
        torch.cuda.empty_cache()
    with open(os.path.join(args.out_dir, "bench_nn_descent.json"), "w") as f:
        json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
