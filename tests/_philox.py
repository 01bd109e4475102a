"""numpy restatement of the keyed draws of o3d_keyed_uniform (csrc/track_eval.cu): Philox4x32-10 with cuRAND's constants,
key = (seed, tracklet id), counter = (element // 4, frame, stream, 0), word element % 4 -> (w >> 8) * 2**-24."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr (..., 4) uint32, key (..., 2) uint32 -> (..., 4) uint32."""
    c = [np.asarray(ctr[..., i], dtype=np.uint32) for i in range(4)]
    k0, k1 = np.asarray(key[..., 0], dtype=np.uint32), np.asarray(key[..., 1], dtype=np.uint32)
    with np.errstate(over="ignore"):
        for r in range(10):
            if r:
                k0, k1 = k0 + W0, k1 + W1
            p0 = M0 * c[0].astype(np.uint64)
            p1 = M1 * c[2].astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & _LO).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & _LO).astype(np.uint32)
            c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return np.stack(c, -1)


def keyed_uniform(seed, tracklet, frame, stream, n):
    """(n,) float32 draws of one slot's stream."""
    e = np.arange(n)
    blocks = np.arange((n + 3) // 4, dtype=np.uint32)
    ctr = np.stack([blocks, np.full_like(blocks, np.uint32(frame & 0xFFFFFFFF)), np.full_like(blocks, stream),
                    np.zeros_like(blocks)], -1)
    key = np.broadcast_to(np.array([seed & 0xFFFFFFFF, tracklet & 0xFFFFFFFF], dtype=np.uint32), (len(blocks), 2))
    words = philox4x32_10(ctr, key).reshape(-1)[:n] if n else np.zeros(0, np.uint32)
    return ((words[e] >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)).astype(np.float32)
