"""Pure-Python restatement of the cross-encoder's dropout keep rule (regtr_b200/csrc/philox.cuh): the masks the
kernels regenerate, for the host tests and the GPU tests to compare against.

Philox4x32-10 with key (seed lo, seed hi) and counter
    (row group << 16 | column,  2^31 | cloud << 11 | layer << 7 | site << 4 | head,  step lo,  step hi)
with cloud = 2 (pair_base + b) + side the global cloud index and row group = row // 8.  Row r of the group reads
half (r & 1) of output word r >> 1; it is kept when that 16-bit value is >= round(p 65536)."""
import numpy as np

M32 = np.uint64(0xFFFFFFFF)
SITES = (1, 2, 3, 4, 5, 6)


def philox(c, k0, k1):
    """Philox4x32-10 over arrays: c = (c0, c1, c2, c3) (broadcastable uint32-valued arrays) -> 4 uint64 arrays."""
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint64) for x in c)
    k0, k1 = np.uint64(k0), np.uint64(k1)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
        k0 = (k0 + np.uint64(0x9E3779B9)) & M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & M32
    return c0, c1, c2, c3


def threshold(p):
    return int(round(float(p) * 65536.0))


def scale(p):
    return np.float32(1.0 / (1.0 - float(p)))


def global_cloud(local, pair_base, n_pairs):
    """Local cloud c of a (src x B, tgt x B) stack -> 2 (pair_base + c % B) + c // B."""
    return 2 * (pair_base + local % n_pairs) + local // n_pairs


def word1(cloud, layer, site, head):
    return (1 << 31) | (int(cloud) << 11) | (int(layer) << 7) | (int(site) << 4) | int(head)


def draws16(seed, step, cloud, layer, site, head, rows, cols):
    """(rows, cols) uint16 draws of a global cloud at one (layer, site, head)."""
    r = np.arange(rows, dtype=np.uint64)[:, None]
    j = np.arange(cols, dtype=np.uint64)[None, :]
    c0 = ((r >> np.uint64(3)) << np.uint64(16)) | j
    w = philox((c0, word1(cloud, layer, site, head), step & 0xFFFFFFFF, (step >> 32) & 0xFFFFFFFF),
               seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    sel = (r & np.uint64(7)) >> np.uint64(1)
    word = np.where(sel == 0, w[0], np.where(sel == 1, w[1], np.where(sel == 2, w[2], w[3])))
    half = np.where((r & np.uint64(1)) == 1, word >> np.uint64(16), word & np.uint64(0xFFFF))
    return half.astype(np.uint16)


def keep_mask(p, seed, step, cloud, layer, site, head, rows, cols):
    """(rows, cols) bool keep mask of global cloud `cloud`."""
    return draws16(seed, step, cloud, layer, site, head, rows, cols) >= threshold(p)


def local_keep_mask(p, seed, step, pair_base, n_pairs, local, layer, site, head, rows, cols):
    return keep_mask(p, seed, step, global_cloud(local, pair_base, n_pairs), layer, site, head, rows, cols)
