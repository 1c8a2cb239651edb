"""Host mirror of the device dropout generator (uniter_b200/csrc/ptx.cuh), vectorised in numpy.

Every dropout site draws its mask from Philox-4x32-10 as a pure function of (seed, stream,
element index): element e uses the counter block e >> 3, counter words (lo(e >> 3), hi(e >> 3),
stream_lo, stream_hi), key (seed_lo, seed_hi), and the 16-bit half (e & 1) of word (e & 7) >> 1 of
the 128-bit output.  An element is dropped iff that 16-bit value is below the threshold of
`dropout_params`.  With a device-side offset `counter` (CUDA-graph replay) the stream becomes
stream + (counter << 20) mod 2^64.

The attention-probability mask keys element (b, h, q, key) as
e = ((b * nheads + h) * 512 + q) * 512 + key; the other sites use e = row * ncols + col.
"""
import numpy as np

ATTN_MAXSEQ = 512          # dropout index pitch of attention (max_position_embeddings)

_M32 = np.uint64(0xFFFFFFFF)
_PHILOX_M0, _PHILOX_M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_PHILOX_W0, _PHILOX_W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)


def philox4x32(c0, c1, c2, c3, k0, k1):
    """Philox-4x32-10 of counter (c0, c1, c2, c3) under key (k0, k1); arrays broadcast.
    Returns the four output words as uint32 arrays."""
    c0, c1, c2, c3, k0, k1 = (np.asarray(x, dtype=np.uint64) & _M32 for x in (c0, c1, c2, c3, k0, k1))
    for _ in range(10):
        p0 = _PHILOX_M0 * c0
        p1 = _PHILOX_M1 * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32
        k0 = (k0 + _PHILOX_W0) & _M32
        k1 = (k1 + _PHILOX_W1) & _M32
    return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def stream_with_offset(stream, counter=None):
    """The stream a kernel uses when it is also given the device offset `counter`."""
    s = int(stream) % (1 << 64)
    if counter is not None:
        s = (s + (int(counter) << 20)) % (1 << 64)
    return s


def rand16(seed, stream, e):
    """The 16-bit random value the device draws for element index e (int array) under (seed, stream)."""
    e = np.asarray(e, dtype=np.uint64)
    g = e >> np.uint64(3)
    seed, stream = int(seed) % (1 << 64), int(stream) % (1 << 64)
    words = np.stack(philox4x32(g & _M32, g >> np.uint64(32), stream & 0xFFFFFFFF, stream >> 32,
                                seed & 0xFFFFFFFF, seed >> 32))
    lane = (e & np.uint64(7)).astype(np.int64)
    w = np.take_along_axis(words, (lane >> 1)[None], 0)[0]
    return np.where(lane & 1, w >> np.uint32(16), w & np.uint32(0xFFFF)).astype(np.uint32)


def dropout_params(p):
    """(threshold, 1 / keep probability) of the kernels for drop probability p: drop iff rand16 < thr;
    kept values are scaled by inv_keep = 65536 / (65536 - thr), computed in fp32 as the device does."""
    t = np.float32(p) * np.float32(65536.0) + np.float32(0.5)
    thr = min(max(int(t), 1), 65535)
    return thr, float(np.float32(65536.0) / np.float32(65536 - thr))


def attn_keep(seed, stream, p, nheads, b, h, nq, nk=None):
    """Boolean keep mask [..., nq, nk] of the attention probabilities of sequence b, head(s) h
    (an int or an int array; rows = queries, columns = keys)."""
    nk = nq if nk is None else nk
    thr, _ = dropout_params(p)
    bh = (np.uint64(b) * np.uint64(nheads) + np.asarray(h, dtype=np.uint64))[..., None, None]
    q = np.arange(nq, dtype=np.uint64)[:, None]
    key = np.arange(nk, dtype=np.uint64)[None]
    e = (bh * np.uint64(ATTN_MAXSEQ) + q) * np.uint64(ATTN_MAXSEQ) + key
    return rand16(seed, stream, e) >= thr
