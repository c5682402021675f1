"""cuvs_b200 — H100-native (sm_90a) scan + top-k kernels behind the cuVS C ABI.

The package layout mirrors the reference's Python binding (python/cuvs/cuvs): ``common`` (Resources),
``neighbors.{brute_force,ivf_flat,ivf_pq,cagra,refine}``, ``cluster.kmeans``, ``preprocessing.quantize.{scalar,binary}``,
``distance``.  Every
function goes through the in-tree ``lib/libcuvs_c.so``; there is no PyTorch or CPU compute fallback.
"""
__version__ = "26.08.00+b200.r1"
