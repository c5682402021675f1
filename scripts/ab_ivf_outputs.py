#!/usr/bin/env python
"""Bit-for-bit comparison of IVF-Flat or IVF-PQ searches and index builds between two builds of the library.

    python scripts/ab_ivf_outputs.py {flat|pq} build DIR
    CUVS_B200_LIB=A/libcuvs_c.so python scripts/ab_ivf_outputs.py {flat|pq} run DIR OUT_A.json [KS]
    CUVS_B200_LIB=B/libcuvs_c.so python scripts/ab_ivf_outputs.py {flat|pq} run DIR OUT_B.json [KS]
    python scripts/ab_ivf_outputs.py {flat|pq} compare OUT_A.json OUT_B.json

    CUVS_B200_LIB=A/libcuvs_c.so python scripts/ab_ivf_outputs.py {flat|pq} build-files DIR_A
    CUVS_B200_LIB=B/libcuvs_c.so python scripts/ab_ivf_outputs.py {flat|pq} build-files DIR_B
    python scripts/ab_ivf_outputs.py {flat|pq} compare-builds DIR_A DIR_B [--by-id]

Searches.  `build` writes seeded indexes to DIR, and both `run`s search the same files, so the comparison covers the search
alone.  `run` writes, per search, one SHA-256 of the neighbours and distances and the number of kernels the library launched
for it (cuvsB200KernelLaunches), or "nondeterministic" when two runs of the search in the same process differ in either.
`compare` lists the searches whose results or launch counts differ and counts those that are nondeterministic in either run.
* flat: dim 128 with 256 lists and dim 96 with 64 lists (the dense coarse select), dim 256 with 128 lists (the streamed-A scan
  kernel) and dim 64 with 4096 lists (the fused coarse select), each in L2, L2 with sqrt, inner product and cosine.  `run`
  searches each at k in {10, 32, 33, 48, 64, 65, 100, 1024, 2048} (the fused top-k path, the 32 < k <= 64 certificate and the
  k > 64 store path; the optional KS, e.g. 100,1024, replaces that list), two batch sizes (only the smaller at k = 2048),
  without and with a bitset filter that keeps 40 % of the rows, and k > 64 once more at the smaller batch under a 1 MB
  workspace budget (CUVS_B200_FLAT_LARGE_K_BUDGET_MB) that splits it.
* pq: indexes that reach every fine-scan path: code stream only; code stream + decoded-row cache (probed densely by the larger
  batch); per-cluster codebooks; pq_bits 5; conservative_memory_allocation, which keeps no decoded rows.  Each comes in L2,
  inner product and cosine.  `run` searches each with CUVS_B200_PQ_PATH unset / lut / stream, the LUT / distance dtypes
  f32/f32, f16/f32, u8/f32 and f16/f16, k in {10, 32, 33, 64, 65, 100, 2048}, two batch sizes (different stream-kernel
  groups), and k > 64 once more under a 1 MB workspace budget (CUVS_B200_PQ_LARGE_K_BUDGET_MB) that splits the batch.

Builds.  `build-files` builds every index above twice in each of three ways: from the dataset on the device, from the same
dataset on the host, and as an empty build extended twice with ids 0..n-1.  It saves each one.  `compare-builds` checks that
the two files of each build in each directory are byte-identical and reports every file that differs between the
directories.  With --by-id, files are compared with each list's (id, payload) rows sorted by id, for a library that does not
keep the rows of a list in input order; everything else in the file must still be identical.
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# name: (dim, build parameters, CUVS_B200_PQ_DECODED_BUDGET_MB when the index is built or loaded)
INDEXES = {
    "flat": {
        "d128": (128, dict(n_lists=256), None),
        "d96": (96, dict(n_lists=64), None),
        "d256": (256, dict(n_lists=128), None),
        "fused_coarse": (64, dict(n_lists=4096), None),
    },
    "pq": {
        "stream":       (128, dict(n_lists=256, pq_dim=64), "0"),
        "stream_d64":   (64, dict(n_lists=256, pq_dim=32), "0"),
        "stream_rows":  (128, dict(n_lists=64, pq_dim=64), None),
        "per_cluster":  (128, dict(n_lists=256, pq_dim=64, codebook_kind="cluster"), None),
        "pq_bits5":     (128, dict(n_lists=256, pq_dim=64, pq_bits=5), None),
        "conservative": (128, dict(n_lists=256, pq_dim=64, conservative_memory_allocation=True), None),
    },
}
METRICS = {"flat": ("sqeuclidean", "euclidean", "inner_product", "cosine"), "pq": ("sqeuclidean", "inner_product", "cosine")}
KS = {"flat": (10, 32, 33, 48, 64, 65, 100, 1024, 2048), "pq": (10, 32, 33, 64, 65, 100, 2048)}
PQ_DTYPES = {"f32": ("float32", "float32"), "f16": ("float16", "float32"), "u8": ("uint8", "float32"), "f16_f16": ("float16", "float16")}
N_ROWS = 60_000
WAYS = ("device", "host", "extend")


def _mod(kind):
    from cuvs_b200.neighbors import ivf_flat, ivf_pq
    return ivf_flat if kind == "flat" else ivf_pq


def _set_env(name, value):
    if value is None:
        os.environ.pop(name, None)
    else:
        os.environ[name] = value


def _data(dim, device=True):
    import numpy as np
    import torch
    rng = np.random.default_rng(7)
    centres = rng.standard_normal((200, dim)).astype(np.float32) * 3
    x = centres[rng.integers(0, 200, N_ROWS)] + rng.standard_normal((N_ROWS, dim)).astype(np.float32)
    q = centres[rng.integers(0, 200, 3000)] + rng.standard_normal((3000, dim)).astype(np.float32)
    x, q = torch.from_numpy(x), torch.from_numpy(q)
    return (x.cuda(), q.cuda()) if device else (x, q)


def _build(kind, metric, name, way="device"):
    import torch
    m = _mod(kind)
    dim, bp, budget = INDEXES[kind][name]
    _set_env("CUVS_B200_PQ_DECODED_BUDGET_MB", budget)
    x = _data(dim, device=way != "host")[0]
    p = dict(metric=metric, kmeans_n_iters=10, **bp)
    if way != "extend":
        idx = m.build(m.IndexParams(**p), x)
    else:
        idx = m.build(m.IndexParams(add_data_on_build=False, **p), x)
        ids = torch.arange(N_ROWS, dtype=torch.int64, device=x.device)
        m.extend(idx, x[:N_ROWS // 3], ids[:N_ROWS // 3])
        m.extend(idx, x[N_ROWS // 3:], ids[N_ROWS // 3:])
    _set_env("CUVS_B200_PQ_DECODED_BUDGET_MB", None)
    return idx


def build(kind, d):
    os.makedirs(d, exist_ok=True)
    for metric in METRICS[kind]:
        for name in INDEXES[kind]:
            _mod(kind).save(os.path.join(d, f"{metric}_{name}.bin"), _build(kind, metric, name))


def build_files(kind, d):
    os.makedirs(d, exist_ok=True)
    for metric in METRICS[kind]:
        for name in INDEXES[kind]:
            print(f"{metric} {name}", flush=True)
            for way in WAYS:
                for rep in (0, 1):
                    _mod(kind).save(os.path.join(d, f"{metric}_{name}_{way}_{rep}.bin"), _build(kind, metric, name, way))


def _launches():
    import ctypes
    from cuvs_b200._capi import lib
    lib.cuvsB200KernelLaunches.restype = ctypes.c_longlong
    return int(lib.cuvsB200KernelLaunches())


def _record(search):
    """-> "<SHA-256 of the distances and neighbours> launches=<kernel launches>" of search(), or "nondeterministic" when two
    calls return different results.  The launches are the second call's: the first may also do one-time work, such as the
    flat code layout the first LUT-kernel search of an IVF-PQ index builds."""
    import torch
    seen, n = set(), 0
    for _ in range(2):
        n0 = _launches()
        dist, i = search()
        torch.cuda.synchronize()
        n = _launches() - n0
        seen.add(hashlib.sha256(dist.cpu().numpy().tobytes() + i.cpu().numpy().tobytes()).hexdigest())
    return f"{seen.pop()} launches={n}" if len(seen) == 1 else "nondeterministic"


def _run_flat(d, ks):
    import numpy as np
    import torch
    from cuvs_b200.neighbors import filters, ivf_flat
    keep = np.random.default_rng(11).random(N_ROWS) < 0.4
    words = np.packbits(np.concatenate([keep, np.zeros((-N_ROWS) % 32, bool)]), bitorder="little").view(np.int32)
    bits = filters.from_bitset(torch.from_numpy(words).cuda())
    res = {}
    for metric in METRICS["flat"]:
        for name, (dim, _, _) in INDEXES["flat"].items():
            idx = ivf_flat.load(os.path.join(d, f"{metric}_{name}.bin"))
            q = _data(dim)[1]
            sp = ivf_flat.SearchParams(n_probes=16)
            print(f"{metric} {name}", flush=True)
            for k in ks:
                for nq in ((300,) if k == 2048 else (300, 3000)):
                    for split in ((False, True) if k > 64 and nq == 300 else (False,)):
                        _set_env("CUVS_B200_FLAT_LARGE_K_BUDGET_MB", "1" if split else None)
                        for filtered in (False, True):
                            f = bits if filtered else None
                            key = f"{metric}/{name}/k={k}/nq={nq}/filtered={filtered}" + ("/split=True" if split else "")
                            res[key] = _record(lambda: ivf_flat.search(sp, idx, q[:nq], k, filter=f))
            _set_env("CUVS_B200_FLAT_LARGE_K_BUDGET_MB", None)
    return res


def _run_pq(d, ks):
    import numpy as np
    from cuvs_b200.neighbors import ivf_pq
    res = {}
    for metric in METRICS["pq"]:
        for name, (dim, _, budget) in INDEXES["pq"].items():
            _set_env("CUVS_B200_PQ_DECODED_BUDGET_MB", budget)
            idx = ivf_pq.load(os.path.join(d, f"{metric}_{name}.bin"))
            _set_env("CUVS_B200_PQ_DECODED_BUDGET_MB", None)
            q = _data(dim)[1]
            print(f"{metric} {name}: streamed={idx.streamed} decoded_rows={idx.has_decoded_rows}", flush=True)
            for env in (None, "lut", "stream"):
                _set_env("CUVS_B200_PQ_PATH", env)
                for dt, (lut, idt) in PQ_DTYPES.items():
                    sp = ivf_pq.SearchParams(n_probes=16, lut_dtype=getattr(np, lut), internal_distance_dtype=getattr(np, idt))
                    for k in ks:
                        for nq in ((300,) if k == 2048 else (300, 3000)):
                            for split in ((False, True) if k > 64 else (False,)):
                                _set_env("CUVS_B200_PQ_LARGE_K_BUDGET_MB", "1" if split else None)
                                res[f"{metric}/{name}/path={env}/{dt}/k={k}/nq={nq}/split={split}"] = \
                                    _record(lambda: ivf_pq.search(sp, idx, q[:nq], k))
            _set_env("CUVS_B200_PQ_PATH", None)
            _set_env("CUVS_B200_PQ_LARGE_K_BUDGET_MB", None)
    return res


def run(kind, d, out_path, ks):
    res = (_run_flat if kind == "flat" else _run_pq)(d, ks)
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


def _by_id_view(kind, path):
    """-> the file's records with each list's rows sorted by id.  Both formats store a list as a count, then (count > 0) its
    payload in groups of 32 rows and its ids: flat f4 [cap, dim] as [cap/32, dim/veclen, 32, veclen], pq (interleaved codes)
    u1 as [groups, chunks, 32, 16]."""
    import numpy as np
    with open(path, "rb") as f:
        if kind == "flat":
            f.read(4)  # dtype tag
        size = os.fstat(f.fileno()).st_size
        recs = []
        while f.tell() < size:
            recs.append(np.lib.format.read_array(f, allow_pickle=False))
    if kind == "flat":
        n_lists, dim = int(recs[3]), int(recs[2])
        head = 10 if bool(recs[8]) else 9  # center norms follow has_norms for L2
    else:
        n_lists, dim, head = int(recs[9]), 0, 14
        assert int(recs[8]) == 1, "only the interleaved code layout is handled"
    sizes, out, r = recs[head].astype(np.int64), recs[:head + 1], head + 1
    for l in range(n_lists):
        count = int(recs[r])
        out.append(recs[r])
        r += 1
        if count == 0:
            continue
        payload, ids = recs[r], recs[r + 1]
        r += 2
        b = (4 if dim % 4 == 0 else 1) if kind == "flat" else 16
        groups = (count + 31) // 32
        rows = payload.reshape(groups, -1, 32, b).transpose(0, 2, 1, 3).reshape(groups * 32, -1)[:sizes[l]]
        order = np.argsort(ids[:sizes[l]], kind="stable")
        out += [rows[order], ids[:sizes[l]][order]]
    assert r == len(recs)
    return out


def compare_builds(kind, da, db, by_id):
    import numpy as np
    names = sorted(n for n in os.listdir(da) if n.endswith(".bin"))
    assert names == sorted(n for n in os.listdir(db) if n.endswith(".bin")), "the directories hold different files"
    read = lambda d, n: open(os.path.join(d, n), "rb").read()
    unstable = [f"{d}/{n}" for d in (da, db) for n in names if n.endswith("_0.bin") and read(d, n) != read(d, n[:-6] + "_1.bin")]
    for u in unstable:
        print("NOT REPRODUCIBLE", u)
    differ = []
    for n in names:
        if by_id:
            va, vb = _by_id_view(kind, os.path.join(da, n)), _by_id_view(kind, os.path.join(db, n))
            same = len(va) == len(vb) and all(np.array_equal(x, y) for x, y in zip(va, vb))
        else:
            same = read(da, n) == read(db, n)
        if not same:
            differ.append(n)
            print("DIFFERS", n)
    print(f"{len(names)} files, {len(differ)} differ{' by id' if by_id else ''}, {len(unstable)} not reproducible within a build")
    return 1 if differ or (unstable and not by_id) else 0


if __name__ == "__main__":
    args = sys.argv[1:]
    if len(args) < 2 or args[0] not in ("flat", "pq"):
        sys.exit(__doc__)
    kind, mode, rest = args[0], args[1], args[2:]
    if mode not in ("compare", "compare-builds"):
        import torch
        if not torch.cuda.is_available():
            sys.exit("ab_ivf_outputs.py builds and searches on the GPU and found none")
    if mode == "build" and len(rest) == 1:
        build(kind, rest[0])
    elif mode == "build-files" and len(rest) == 1:
        build_files(kind, rest[0])
    elif mode == "run" and len(rest) in (2, 3):
        run(kind, rest[0], rest[1], tuple(int(k) for k in rest[2].split(",")) if len(rest) == 3 else KS[kind])
    elif mode == "compare" and len(rest) == 2:
        sys.exit(compare(*rest))
    elif mode == "compare-builds" and len(rest) in (2, 3) and rest[2:] in ([], ["--by-id"]):
        sys.exit(compare_builds(kind, rest[0], rest[1], rest[2:] == ["--by-id"]))
    else:
        sys.exit(__doc__)
