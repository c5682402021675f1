"""IVF-PQ code rows as `list_data` and `transform` return them, turned into one code per byte.

A row holds pq_dim codes of pq_bits bits packed contiguously, least significant bit first, in ceil(pq_dim * pq_bits / 8)
bytes: code j occupies bits [j * pq_bits, (j + 1) * pq_bits) of the row read as one little-endian integer, so for
pq_bits < 8 a code may straddle two bytes (the reference's bitfield_ref_t order,
cpp/src/neighbors/ivf_pq/ivf_pq_codepacking.cuh:30-55).  NumPy only: the CPU tests import it."""
import numpy as np


def row_bytes(pq_dim, pq_bits):
    return (pq_dim * pq_bits + 7) // 8


def unpack_codes(packed, pq_dim, pq_bits):
    """[n, row_bytes] uint8 -> [n, pq_dim] uint8 codes."""
    packed = np.asarray(packed, np.uint8)
    n, ld = packed.shape
    assert ld == row_bytes(pq_dim, pq_bits), (ld, pq_dim, pq_bits)
    bits = np.unpackbits(packed, axis=1, bitorder="little")[:, :pq_dim * pq_bits].reshape(n, pq_dim, pq_bits)
    return (bits.astype(np.uint16) << np.arange(pq_bits, dtype=np.uint16)).sum(-1).astype(np.uint8)


def index_codes(index):
    """-> (list offsets [n_lists + 1], codes [n, pq_dim] one per byte, ids [n]) of a built index, lists concatenated."""
    sizes = index.list_sizes.cpu().numpy().astype(np.int64)
    offs = np.concatenate([[0], np.cumsum(sizes)])
    pq_dim, pq_bits = index.pq_dim, index.pq_bits
    codes = [np.zeros((0, pq_dim), np.uint8)]
    ids = [np.zeros(0, np.int64)]
    for l in range(index.n_lists):
        if sizes[l]:
            codes.append(unpack_codes(index.list_data(l).cpu().numpy(), pq_dim, pq_bits))
            ids.append(index.list_indices(l).cpu().numpy())
    return offs, np.concatenate(codes), np.concatenate(ids)
