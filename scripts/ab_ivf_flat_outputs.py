#!/usr/bin/env python
"""Bit-for-bit comparison of IVF-Flat search results between two builds of the library.

    python scripts/ab_ivf_flat_outputs.py build DIR
    CUVS_B200_LIB=A/libcuvs_c.so python scripts/ab_ivf_flat_outputs.py run DIR OUT_A.json
    CUVS_B200_LIB=B/libcuvs_c.so python scripts/ab_ivf_flat_outputs.py run DIR OUT_B.json
    python scripts/ab_ivf_flat_outputs.py compare OUT_A.json OUT_B.json

`build` writes seeded indexes to DIR: dim 128 with 256 lists and dim 96 with 64 lists (the dense coarse select), dim 256 with
128 lists (the streamed-A scan kernel) and dim 64 with 4096 lists (the fused coarse select).  Each comes in L2, L2 with sqrt,
inner product and cosine.  Both runs load the same files, because a build may place the rows of a list in a different order,
and equal distances are ordered by that position.  `run` searches each index at k in {10, 32, 64} (the fused top-k path; an
optional last argument, e.g. 100,1024, replaces that list), two batch sizes, without and with a bitset filter that keeps 40 %
of the rows.  It writes one
SHA-256 of the neighbours and distances per search, or "nondeterministic" when two runs of the search in the same process
differ.  `compare` lists the searches whose results differ and counts those that are nondeterministic in either run.
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

INDEXES = {  # name: (dim, n_lists)
    "d128": (128, 256),
    "d96": (96, 64),
    "d256": (256, 128),
    "fused_coarse": (64, 4096),
}
METRICS = ("sqeuclidean", "euclidean", "inner_product", "cosine")
KS = (10, 32, 64)
N_ROWS = 60_000


def _data(dim):
    import numpy as np
    import torch
    rng = np.random.default_rng(7)
    centres = rng.standard_normal((200, dim)).astype(np.float32) * 3
    x = centres[rng.integers(0, 200, N_ROWS)] + rng.standard_normal((N_ROWS, dim)).astype(np.float32)
    q = centres[rng.integers(0, 200, 3000)] + rng.standard_normal((3000, dim)).astype(np.float32)
    return torch.from_numpy(x).cuda(), torch.from_numpy(q).cuda()


def _bitset():
    import numpy as np
    import torch
    from cuvs_b200.neighbors import filters
    keep = np.random.default_rng(11).random(N_ROWS) < 0.4
    bits = np.packbits(np.concatenate([keep, np.zeros((-N_ROWS) % 32, bool)]), bitorder="little").view(np.int32)
    return filters.from_bitset(torch.from_numpy(bits).cuda())


def build(d):
    from cuvs_b200.neighbors import ivf_flat
    os.makedirs(d, exist_ok=True)
    for metric in METRICS:
        for name, (dim, n_lists) in INDEXES.items():
            p = ivf_flat.IndexParams(n_lists=n_lists, metric=metric, kmeans_n_iters=10)
            ivf_flat.save(os.path.join(d, f"{metric}_{name}.bin"), ivf_flat.build(p, _data(dim)[0]))


def run(d, out_path, ks=KS):
    import torch
    from cuvs_b200.neighbors import ivf_flat

    def digest(sp, idx, q, k, filt):
        dist, i = ivf_flat.search(sp, idx, q, k, filter=filt)
        torch.cuda.synchronize()
        return hashlib.sha256(dist.cpu().numpy().tobytes() + i.cpu().numpy().tobytes()).hexdigest()

    res = {}
    bits = _bitset()
    for metric in METRICS:
        for name, (dim, _) in INDEXES.items():
            idx = ivf_flat.load(os.path.join(d, f"{metric}_{name}.bin"))
            q = _data(dim)[1]
            sp = ivf_flat.SearchParams(n_probes=16)
            print(f"{metric} {name}", flush=True)
            for k in ks:
                for nq in (300, 3000):
                    for filtered in (False, True):
                        h = {digest(sp, idx, q[:nq], k, bits if filtered else None) for _ in range(2)}
                        res[f"{metric}/{name}/k={k}/nq={nq}/filtered={filtered}"] = h.pop() if len(h) == 1 else "nondeterministic"
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
        sys.exit("ab_ivf_flat_outputs.py searches on the GPU and found none")
    if len(sys.argv) == 3 and sys.argv[1] == "build":
        build(sys.argv[2])
    elif len(sys.argv) in (4, 5) and sys.argv[1] == "run":
        run(sys.argv[2], sys.argv[3], tuple(int(k) for k in sys.argv[4].split(",")) if len(sys.argv) == 5 else KS)
    elif len(sys.argv) == 4 and sys.argv[1] == "compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    else:
        sys.exit(__doc__)
