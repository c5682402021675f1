#!/usr/bin/env python
"""The scalar and binary quantizers over 10M x 768 embedding rows on the device, against the HBM bound.

    python scripts/bench_quantize.py --out-dir DIR [--n 10000000] [--d 768] [--rounds 3] [--host-rows 1000000]

Rows come from bench.py's embedding-like manifold generator, in float32 and then float16 (one type on the device at a time).
For each type the script times, with CUDA events after a warm-up call of each, over --rounds rounds that alternate the calls:
  - binary transform with threshold ZERO and with a trained MEAN threshold row;
  - scalar transform (rows to int8 codes) and its inverse (codes to rows of the same type);
  - the torch composition that packs `x > 0` by bit weights (the way scripts/bench_cagra_hamming.py packs its rows, most
    significant bit first), in 1M-row chunks;
  - each train: binary MEAN, binary SAMPLING_MEDIAN at ratio 0.1 and scalar at quantile 0.99.
For each transform it prints the bytes read plus written, the least time those bytes take at 3.35 TB/s (the H100 SXM's
HBM3 data-sheet bandwidth) and the share of that bound reached (best round).  It also times a --host-rows binary and scalar
transform of pinned host rows (copies over PCIe included).  The card's name and power limit are read in the same run.
Everything goes to stdout and to DIR/bench_quantize.json.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from bench import gen_manifold  # noqa: E402
from bench_ivf_pq_cosine import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def timed(fn):
    """(result, ms) of one call between CUDA events on the current stream."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return out, a.elapsed_time(b)


def torch_sign_pack(x, chunk=1 << 20):
    """(x > 0) packed eight columns to a byte by bit weights, most significant first (uint8 [n, d / 8])."""
    n, d = x.shape
    weights = (2 ** torch.arange(7, -1, -1, device=x.device)).to(torch.uint8)
    out = torch.empty((n, d // 8), dtype=torch.uint8, device=x.device)
    for s in range(0, n, chunk):
        e = min(n, s + chunk)
        b = (x[s:e] > 0).to(torch.uint8).view(e - s, d // 8, 8)
        out[s:e] = (b * weights).sum(-1, dtype=torch.uint8)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out-dir", required=True)
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--host-rows", type=int, default=1_000_000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_quantize needs a CUDA device"
    from cuvs_b200.common.resources import Resources
    from cuvs_b200.preprocessing.quantize import binary, scalar

    os.makedirs(args.out_dir, exist_ok=True)
    n, d = args.n, args.d
    res = Resources()
    result = {"card": card(0), "n": n, "d": d, "rounds": args.rounds, "hbm_bound_bytes_per_s": HBM_BYTES_PER_S, "types": {}}
    for tname, dt in (("float32", torch.float32), ("float16", torch.float16)):
        x = gen_manifold(n, d, seed=5).to(dt)
        esz = x.element_size()
        nb = (d + 7) // 8
        trains = {
            "binary MEAN": lambda: binary.train(binary.QuantizerParams(threshold="mean"), x, resources=res),
            "binary SAMPLING_MEDIAN 0.1": lambda: binary.train(binary.QuantizerParams(threshold="sampling_median", sampling_ratio=0.1), x,
                                                               resources=res),
            "scalar 0.99": lambda: scalar.train(scalar.QuantizerParams(quantile=0.99), x, resources=res),
        }
        mean_q = trains["binary MEAN"]()
        sq = trains["scalar 0.99"]()
        bits = torch.empty((n, nb), dtype=torch.uint8, device="cuda")
        codes = torch.empty((n, d), dtype=torch.int8, device="cuda")
        back = torch.empty((n, d), dtype=dt, device="cuda")
        calls = {
            "binary transform ZERO": (lambda: binary.transform(x, output=bits, resources=res), n * d * esz + n * nb),
            "binary transform MEAN": (lambda: binary.transform(x, output=bits, quantizer=mean_q, resources=res), n * d * esz + n * nb),
            "scalar transform": (lambda: scalar.transform(sq, x, output=codes, resources=res), n * d * esz + n * d),
            "scalar inverse": (lambda: scalar.inverse_transform(sq, codes, output=back, resources=res), n * d + n * d * esz),
            "torch (x > 0) packed by weights": (lambda: torch_sign_pack(x), n * d * esz + n * nb),
        }
        times = {k: [] for k in list(calls) + list(trains)}
        for fn, _ in calls.values():  # warm-up
            fn()
        for fn in trains.values():
            fn()
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for k, (fn, _) in calls.items():
                times[k].append(timed(fn)[1])
            for k, fn in trains.items():
                times[k].append(timed(fn)[1])
        rows = {}
        for k, ms in times.items():
            entry = {"ms": [round(v, 3) for v in ms], "best_ms": round(min(ms), 3)}
            if k in calls:
                nbytes = calls[k][1]
                bound_ms = nbytes / HBM_BYTES_PER_S * 1e3
                entry.update(bytes=nbytes, bound_ms=round(bound_ms, 3), share_of_bound=round(bound_ms / min(ms), 3))
            rows[k] = entry
            extra = f"  {entry['bytes'] / 1e9:.2f} GB, bound {entry['bound_ms']:.2f} ms, {100 * entry['share_of_bound']:.1f}% of it" \
                if "bytes" in entry else ""
            print(f"{tname:8s} {k:34s} {', '.join(f'{v:.2f}' for v in ms)} ms{extra}", flush=True)
        result["types"][tname] = rows
        del x, bits, codes, back, mean_q
        torch.cuda.empty_cache()

    # pinned host rows: the library streams them through device buffers (copies over PCIe included)
    hx = gen_manifold(args.host_rows, d, seed=6).cpu().pin_memory()
    hbits = torch.empty((args.host_rows, (d + 7) // 8), dtype=torch.uint8).pin_memory()
    hcodes = torch.empty((args.host_rows, d), dtype=torch.int8).pin_memory()
    hq = scalar.train(scalar.QuantizerParams(quantile=0.99), hx, resources=res)
    host = {}
    for k, fn in (("binary transform ZERO", lambda: binary.transform(hx, output=hbits, resources=res)),
                  ("scalar transform", lambda: scalar.transform(hq, hx, output=hcodes, resources=res))):
        fn()
        ms = []
        for _ in range(args.rounds):
            t0 = time.perf_counter()
            fn()  # returns once the host output is written
            ms.append((time.perf_counter() - t0) * 1e3)
        host[k] = {"ms": [round(v, 3) for v in ms], "rows": args.host_rows}
        print(f"pinned   {k:34s} {', '.join(f'{v:.2f}' for v in ms)} ms ({args.host_rows} rows)", flush=True)
    result["pinned_host"] = host
    print(f"card: {result['card']}")
    with open(os.path.join(args.out_dir, "bench_quantize.json"), "w") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
