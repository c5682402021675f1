"""Time IVF-PQ builds, whose coarse centres are trained by the k-means loop (kmeans_train), and k-means fits on their own.

Usage: python scripts/bench_kmeans_ivf_pq_build.py [--rounds 3] [--out FILE]

Data: a mixture of 1000 Gaussians (centres N(0, I), sigma 0.25) generated on the GPU from a fixed seed.  Shapes:
  ivf_pq_1024: 2M x 128, n_lists 1024, pq_dim 64, 20 k-means iterations on 1M training rows;
  ivf_pq_8192: 4M x 128, n_lists 8192, pq_dim 64, 10 k-means iterations on 2M training rows;
  kmeans_fit:  1M x 128, 1024 clusters, 20 iterations (tol 0), k-means++ seeding;
  kmeans_fit_shift100: the same fit with every component of the data shifted by +100, where the exact assignment's
               certificate rejects most rows and they are scored against every centre.
Each shape is built once to warm up, then `rounds` times; every timing ends in a device synchronise.  Prints one JSON line
with the GPU's name and power limit and, per shape, the build times in seconds.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def mixture(n, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    centres = torch.randn(1000, d, generator=g, device="cuda")
    out = torch.empty(n, d, device="cuda")
    step = 1 << 20
    for r0 in range(0, n, step):
        r1 = min(n, r0 + step)
        lab = torch.randint(0, 1000, (r1 - r0,), generator=g, device="cuda")
        out[r0:r1] = centres[lab] + 0.25 * torch.randn(r1 - r0, d, generator=g, device="cuda")
    return out


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    from cuvs_b200.cluster import kmeans
    from cuvs_b200.neighbors import ivf_pq

    shapes = {
        "ivf_pq_1024": (2_000_000, 128, dict(n_lists=1024, pq_dim=64, kmeans_n_iters=20, kmeans_trainset_fraction=0.5)),
        "ivf_pq_8192": (4_000_000, 128, dict(n_lists=8192, pq_dim=64, kmeans_n_iters=10, kmeans_trainset_fraction=0.5)),
    }
    result = {"gpu": gpu_info(), "rounds": a.rounds, "seconds": {}}
    for name, (n, d, kw) in shapes.items():
        x = mixture(n, d, 1234)
        p = ivf_pq.IndexParams(**kw)
        timed(lambda: ivf_pq.build(p, x))
        result["seconds"][name] = [round(timed(lambda: ivf_pq.build(p, x)), 4) for _ in range(a.rounds)]
        del x
    x = mixture(1_000_000, 128, 99)
    kp = kmeans.KMeansParams(n_clusters=1024, max_iter=20, tol=0.0)
    timed(lambda: kmeans.fit(kp, x))
    result["seconds"]["kmeans_fit"] = [round(timed(lambda: kmeans.fit(kp, x)), 4) for _ in range(a.rounds)]
    x += 100.0
    timed(lambda: kmeans.fit(kp, x))
    result["seconds"]["kmeans_fit_shift100"] = [round(timed(lambda: kmeans.fit(kp, x)), 4) for _ in range(a.rounds)]
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
