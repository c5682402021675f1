#!/usr/bin/env python
"""Bit-for-bit comparison of IVF-PQ search results between two builds of the library.

    python scripts/ab_ivf_pq_outputs.py build DIR
    CUVS_B200_LIB=A/libcuvs_c.so python scripts/ab_ivf_pq_outputs.py run DIR OUT_A.json
    CUVS_B200_LIB=B/libcuvs_c.so python scripts/ab_ivf_pq_outputs.py run DIR OUT_B.json
    python scripts/ab_ivf_pq_outputs.py compare OUT_A.json OUT_B.json

`build` writes seeded indexes to DIR that reach every fine-scan path: code stream only; code stream + decoded-row cache (probed
densely by the larger batch); per-cluster codebooks; pq_bits 5; conservative_memory_allocation, which keeps no decoded rows.
Each comes in L2, inner product and cosine.  Both runs load the same files, because a build may place the rows of a list in a
different order, and equal distances are ordered by that position.  `run` searches each index with CUVS_B200_PQ_PATH unset /
lut / stream, the LUT / distance dtypes f32/f32, f16/f32, u8/f32 and f16/f16, k in {10, 32, 33, 64, 65, 100, 2048}, two
batch sizes (different stream-kernel groups), and k > 64 once more under a 1 MB workspace budget
(CUVS_B200_PQ_LARGE_K_BUDGET_MB) that splits the batch.  It writes one SHA-256 of the neighbours and distances per search,
or "nondeterministic" when two runs of the search in the same process differ.  `compare` lists the searches whose results
differ and counts those that are nondeterministic in either run.
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

INDEXES = {  # name: (dim, build parameters, CUVS_B200_PQ_DECODED_BUDGET_MB when the index is built or loaded)
    "stream":       (128, dict(pq_dim=64), "0"),
    "stream_d64":   (64, dict(pq_dim=32), "0"),
    "stream_rows":  (128, dict(pq_dim=64, n_lists=64), None),
    "per_cluster":  (128, dict(pq_dim=64, codebook_kind="cluster"), None),
    "pq_bits5":     (128, dict(pq_dim=64, pq_bits=5), None),
    "conservative": (128, dict(pq_dim=64, conservative_memory_allocation=True), None),
}
METRICS = ("sqeuclidean", "inner_product", "cosine")
DTYPES = {"f32": ("float32", "float32"), "f16": ("float16", "float32"), "u8": ("uint8", "float32"), "f16_f16": ("float16", "float16")}
KS = (10, 32, 33, 64, 65, 100, 2048)


def _set_env(name, value):
    if value is None:
        os.environ.pop(name, None)
    else:
        os.environ[name] = value


def _data(dim):
    import numpy as np
    import torch
    rng = np.random.default_rng(7)
    centres = rng.standard_normal((200, dim)).astype(np.float32) * 3
    x = centres[rng.integers(0, 200, 60_000)] + rng.standard_normal((60_000, dim)).astype(np.float32)
    q = centres[rng.integers(0, 200, 3000)] + rng.standard_normal((3000, dim)).astype(np.float32)
    return torch.from_numpy(x).cuda(), torch.from_numpy(q).cuda()


def build(d):
    from cuvs_b200.neighbors import ivf_pq
    os.makedirs(d, exist_ok=True)
    for metric in METRICS:
        for name, (dim, bp, budget) in INDEXES.items():
            _set_env("CUVS_B200_PQ_DECODED_BUDGET_MB", budget)
            p = dict(n_lists=256, metric=metric, kmeans_n_iters=10)
            p.update(bp)
            ivf_pq.save(os.path.join(d, f"{metric}_{name}.bin"), ivf_pq.build(ivf_pq.IndexParams(**p), _data(dim)[0]))
    _set_env("CUVS_B200_PQ_DECODED_BUDGET_MB", None)


def run(d, out_path):
    import numpy as np
    import torch
    from cuvs_b200.neighbors import ivf_pq

    def digest(sp, idx, q, k):
        d, i = ivf_pq.search(sp, idx, q, k)
        torch.cuda.synchronize()
        return hashlib.sha256(d.cpu().numpy().tobytes() + i.cpu().numpy().tobytes()).hexdigest()

    res = {}
    for metric in METRICS:
        for name, (dim, _, budget) in INDEXES.items():
            _set_env("CUVS_B200_PQ_DECODED_BUDGET_MB", budget)
            idx = ivf_pq.load(os.path.join(d, f"{metric}_{name}.bin"))
            _set_env("CUVS_B200_PQ_DECODED_BUDGET_MB", None)
            q = _data(dim)[1]
            print(f"{metric} {name}: streamed={idx.streamed} decoded_rows={idx.has_decoded_rows}", flush=True)
            for env in (None, "lut", "stream"):
                _set_env("CUVS_B200_PQ_PATH", env)
                for dt, (lut, idt) in DTYPES.items():
                    sp = ivf_pq.SearchParams(n_probes=16, lut_dtype=getattr(np, lut), internal_distance_dtype=getattr(np, idt))
                    for k in KS:
                        for nq in ((300,) if k == 2048 else (300, 3000)):
                            for split in ((False, True) if k > 64 else (False,)):
                                _set_env("CUVS_B200_PQ_LARGE_K_BUDGET_MB", "1" if split else None)
                                h = {digest(sp, idx, q[:nq], k) for _ in range(2)}
                                res[f"{metric}/{name}/path={env}/{dt}/k={k}/nq={nq}/split={split}"] = \
                                    h.pop() if len(h) == 1 else "nondeterministic"
            _set_env("CUVS_B200_PQ_PATH", None)
            _set_env("CUVS_B200_PQ_LARGE_K_BUDGET_MB", None)
    with open(out_path, "w") as f:
        json.dump(res, f, indent=0, sort_keys=True)
    print(f"{len(res)} searches -> {out_path}")


def compare(a_path, b_path):
    a, b = json.load(open(a_path)), json.load(open(b_path))
    keys = sorted(set(a) | set(b))
    nondet = [k for k in keys if "nondeterministic" in (a.get(k), b.get(k))]
    bad = [k for k in keys if k not in nondet and a.get(k) != b.get(k)]
    for k in nondet:
        print("NONDETERMINISTIC", k)
    for k in bad:
        print("DIFFERS", k)
    print(f"{len(keys)} searches, {len(bad)} differ, {len(nondet)} nondeterministic")
    return 1 if bad else 0


if __name__ == "__main__":
    import torch
    if sys.argv[1:2] != ["compare"] and not torch.cuda.is_available():
        sys.exit("ab_ivf_pq_outputs.py searches on the GPU and found none")
    if len(sys.argv) == 3 and sys.argv[1] == "build":
        build(sys.argv[2])
    elif len(sys.argv) == 4 and sys.argv[1] == "run":
        run(sys.argv[2], sys.argv[3])
    elif len(sys.argv) == 4 and sys.argv[1] == "compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    else:
        sys.exit(__doc__)
