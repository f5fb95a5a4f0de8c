"""CPU: a numpy restatement of Philox4x32-10, the generator behind vima_head_sample's draws, pinned to Random123's known answers.
The GPU tests (test_action_sampling_gpu.py) hold the kernel's uniforms to this restatement."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: uint32 (..., 4), key: uint32 (..., 2) (broadcast) -> uint32 (..., 4)."""
    c = [np.asarray(ctr, dtype=np.uint32)[..., i].astype(np.uint64) for i in range(4)]
    key = np.asarray(key, dtype=np.uint32)
    k0, k1 = key[..., 0].astype(np.uint64), key[..., 1].astype(np.uint64)
    for r in range(10):
        if r:
            k0 = (k0 + np.uint64(W0)) & _LO
            k1 = (k1 + np.uint64(W1)) & _LO
        p0, p1 = M0 * c[0], M1 * c[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & _LO, p1 >> np.uint64(32), p1 & _LO
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return np.stack([x.astype(np.uint32) for x in c], axis=-1)


def head_uniforms(B: int, n_heads: int, seed: int, draw: int) -> np.ndarray:
    """The u of every (row, head) of one sampling launch: float64 [B, n_heads], exactly the kernel's fp32 value."""
    b, h = np.meshgrid(np.arange(B, dtype=np.uint32), np.arange(n_heads, dtype=np.uint32), indexing="ij")
    ctr = np.stack([b, h, np.full_like(b, draw & 0xFFFFFFFF), np.full_like(b, draw >> 32)], axis=-1)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint32)
    return (philox4x32_10(ctr, key)[..., 0] >> np.uint32(8)).astype(np.float64) * 2.0 ** -24


def _hex(words):
    return " ".join(f"{int(w):08x}" for w in words)


def test_known_answers():
    """Random123's kat_vectors for philox4x32_10 (counter, key -> output)."""
    cases = [
        ((0, 0, 0, 0), (0, 0), "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
        ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
        ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), "d16cfe09 94fdcceb 5001e420 24126ea1"),
    ]
    for ctr, key, want in cases:
        assert _hex(philox4x32_10(np.array(ctr, dtype=np.uint32), np.array(key, dtype=np.uint32))) == want


def test_uniforms_are_24_bit_and_in_range():
    u = head_uniforms(64, 12, seed=0x0123456789ABCDEF, draw=(1 << 32) + 5)
    assert u.shape == (64, 12)
    assert (u >= 0).all() and (u < 1).all()
    assert np.array_equal(u * 2 ** 24, np.floor(u * 2 ** 24))
    assert len(np.unique(u)) > 64 * 12 - 5  # distinct streams per (row, head)
    assert not np.array_equal(u, head_uniforms(64, 12, seed=0x0123456789ABCDEF, draw=5))  # the draw's high word is in the counter
