"""NumPy restatement of the texture-synthesis noise (``wctb200_noise_u8``, include/wctb200.h): Philox4x32-10 (Random123),
vectorised over blocks.  Test infrastructure only.

Byte j of frame f (row-major HWC) is byte j % 16 of Philox4x32-10 with counter (b_lo, b_hi, f_lo, f_hi), b = j // 16, and
key (seed_lo, seed_hi); the 16 bytes are x0..x3, each little-endian."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = np.uint64(0xFFFFFFFF)
_32 = np.uint64(32)


def philox4x32_10(counter, key):
    """counter: uint32-valued array [..., 4]; key: (k0, k1) ints.  Returns uint32 [..., 4]."""
    c = [np.asarray(counter, dtype=np.uint64)[..., i] for i in range(4)]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [(p1 >> _32) ^ c[1] ^ np.uint64(k0), p1 & MASK, (p0 >> _32) ^ c[3] ^ np.uint64(k1), p0 & MASK]
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return np.stack(c, axis=-1).astype(np.uint32)


def noise_frame(nbytes, seed, index):
    """The ``nbytes`` bytes of absolute frame ``index``, uint8 [nbytes]."""
    nb = (nbytes + 15) // 16
    b = np.arange(nb, dtype=np.uint64)
    ctr = np.empty((nb, 4), dtype=np.uint64)
    ctr[:, 0], ctr[:, 1] = b & MASK, b >> _32
    ctr[:, 2], ctr[:, 3] = index & 0xFFFFFFFF, index >> 32
    x = philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))
    return x.astype("<u4").view(np.uint8).reshape(-1)[:nbytes]


def noise_u8(count, H, W, C=3, seed=0, first_index=0):
    """uint8 [count, H, W, C]: frames first_index .. first_index + count - 1."""
    return np.stack([noise_frame(H * W * C, seed, first_index + n).reshape(H, W, C) for n in range(count)])
