"""numpy restatement of the library's counter-based noise (csrc/bdiff_philox.cuh, layout in include/bdiff.h): Philox4x32-10
over counter {block lo, block hi, draw lo, draw hi} and key {seed lo, seed hi}, then Box-Muller in float64 rounded to
float32.  Shared by test_native_sample_cpu.py and test_gpu_native_sample.py."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr: np.ndarray, key: np.ndarray) -> np.ndarray:
    """ctr uint32 [n, 4], key uint32 [n, 2] -> uint32 [n, 4]."""
    c = [ctr[:, i].astype(np.uint64) for i in range(4)]
    k0, k1 = key[:, 0].astype(np.uint32), key[:, 1].astype(np.uint32)
    for _ in range(10):
        p0 = M0 * c[0]
        p1 = M1 * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & MASK32
        hi1, lo1 = p1 >> np.uint64(32), p1 & MASK32
        c = [hi1 ^ c[1] ^ k0.astype(np.uint64), lo1, hi0 ^ c[3] ^ k1.astype(np.uint64), lo0]
        k0 = k0 + W0
        k1 = k1 + W1
    return np.stack(c, axis=1).astype(np.uint32)


def blocks(seed: int, draw: int, count: int) -> np.ndarray:
    """The raw words of blocks 0 .. count-1 of draw `draw` of `seed`: uint32 [count, 4]."""
    b = np.arange(count, dtype=np.uint64)
    ctr = np.stack([b & MASK32, b >> np.uint64(32), np.full(count, draw & 0xFFFFFFFF, np.uint64),
                    np.full(count, draw >> 32, np.uint64)], axis=1).astype(np.uint32)
    key = np.tile(np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint32), (count, 1))
    return philox4x32_10(ctr, key)


def normals(seed: int, draw: int, n: int) -> np.ndarray:
    """Elements 0 .. n-1 of draw `draw` of `seed` (float32)."""
    w = blocks(seed, draw, (n + 3) // 4).astype(np.float64)
    r0 = np.sqrt(-2.0 * np.log((w[:, 0] + 0.5) * 2.0 ** -32))
    r1 = np.sqrt(-2.0 * np.log((w[:, 2] + 0.5) * 2.0 ** -32))
    a0, a1 = np.pi * (w[:, 1] * 2.0 ** -31), np.pi * (w[:, 3] * 2.0 ** -31)
    out = np.stack([r0 * np.cos(a0), r0 * np.sin(a0), r1 * np.cos(a1), r1 * np.sin(a1)], axis=1)
    return out.reshape(-1)[:n].astype(np.float32)
