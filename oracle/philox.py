"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the device-RNG streams of v2e_b200/csrc/emu.cu.

rng_mode="device" draws per-frame noise in-kernel from Philox4x32-7 (Salmon et al., SC'11), keyed by the 64-bit seed
(key = (seed low word, seed high word)) and counted by (quad of 4 pixels, Philox frame index, stream, tag):

    leak  (noise_quad)    counter (q, f, 0, 0x6c65616b "leak"), q = whole-frame pixel index >> 2
    shot  (shot_uniform)  counter (q, f, 1, 0x73686f74 "shot"), q as above
    photo (pr_noise_quad) counter (q, f, 2, 0x70726e7a "prnz"), q = the handle's LOCAL pixel index >> 2

Written from the algorithm's definition, independently of the CUDA source, so that a test can hold the device's
dumped draws against it. The shot uniforms are reproduced bit for bit. The normals go through __logf, sqrt.approx and
__sincosf on the device, so only their Box-Muller inputs are restated exactly: the radius argument u (float32) and the
angle (float32), from which radius^2 = -2 ln u and the angle follow.
"""
import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
TAG_LEAK, TAG_SHOT, TAG_PR = 0x6c65616b, 0x73686f74, 0x70726e7a
ROUNDS = 7
_M32 = np.uint64(0xFFFFFFFF)
TWO_PI_F32 = np.float32(6.283185307179586)


def philox4x32(ctr, key, rounds=ROUNDS):
    """Philox4x32-R. ctr: 4 uint32 arrays (broadcastable), key: 2 uint32 scalars / arrays. Returns 4 uint32 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, np.uint64) & _M32 for c in ctr)
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0, k1 = (np.uint64(int(k) & 0xFFFFFFFF) for k in key)
    for _ in range(rounds):
        p0 = np.uint64(M0) * c0             # < 2^64: exact in uint64
        p1 = np.uint64(M1) * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & _M32
        hi1, lo1 = p1 >> np.uint64(32), p1 & _M32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0 = (k0 + np.uint64(W0)) & _M32
        k1 = (k1 + np.uint64(W1)) & _M32
    return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def seed_key(seed):
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return seed & 0xFFFFFFFF, seed >> 32


def _words(seed, quads, frame_index, stream, tag, rounds=ROUNDS):
    q = np.asarray(quads, np.uint64)
    return philox4x32((q, np.full_like(q, frame_index), np.full_like(q, stream), np.full_like(q, tag)),
                      seed_key(seed), rounds)


def _pick(words, j, a, b):
    """Per pixel: word a for pixels 0, 1 of the quad, word b for pixels 2, 3."""
    return np.where(j < 2, words[a], words[b])


def u01_open(x):
    """((x >> 8) + 0.5) * 2^-24, rounded once to float32 (the device's fmaf)."""
    return (((x >> np.uint32(8)).astype(np.float64) + 0.5) * 2.0 ** -24).astype(np.float32)


def u01_half(x):
    return ((x >> np.uint32(8)).astype(np.float64) * 2.0 ** -24).astype(np.float32)


def uint32_to_float_rz(u):
    """__uint2float_rz: uint32 -> float32 rounded toward zero."""
    u = np.asarray(u, np.uint64)
    _, e = np.frexp(u.astype(np.float64))           # u = m * 2^e, m in [0.5, 1): e = bit length
    sh = np.maximum(e - 24, 0).astype(np.uint64)
    return ((u >> sh) << sh).astype(np.float32)     # exactly representable now


def leak_fields(seed, n, frame_index, px_off=0, rounds=ROUNDS):
    """Per pixel of a handle of n pixels: (u, angle, sin_or_cos, pref). The leak normal is
    sqrt(-2 ln u) * (cos(angle) if sin_or_cos == 0 else sin(angle)); pref is the 12-bit prefix of the shot uniform."""
    g = np.arange(n, dtype=np.uint64) + np.uint64(px_off)
    j = (g & np.uint64(3)).astype(np.int64)
    w = _words(seed, g >> np.uint64(2), frame_index, 0, TAG_LEAK, rounds)
    u = u01_open(_pick(w, j, 0, 2))
    ang16 = (_pick(w, j, 1, 3) >> np.uint32(16)).astype(np.float32) * np.float32(1.0 / 65536.0)
    angle = TWO_PI_F32 * ang16
    x, y, z, ww = w
    pref = np.select([j == 0, j == 1, j == 2],
                     [(x & 0xff) | ((y & 0xf) << 8), (y >> 4) & 0xfff, (z & 0xff) | ((ww & 0xf) << 8)],
                     (ww >> 4) & 0xfff).astype(np.uint32)
    return u, angle, (j & 1), pref


def shot_u01(seed, n, frame_index, px_off=0, rounds=ROUNDS):
    """The full shot-noise uniform of every pixel: float_rz((pref << 20) | (w >> 12)) * 2^-32, bit for bit."""
    g = np.arange(n, dtype=np.uint64) + np.uint64(px_off)
    j = (g & np.uint64(3)).astype(np.int64)
    pref = leak_fields(seed, n, frame_index, px_off, rounds)[3]
    w = np.choose(j, _words(seed, g >> np.uint64(2), frame_index, 1, TAG_SHOT, rounds))
    u = (pref.astype(np.uint64) << np.uint64(20)) | (w.astype(np.uint64) >> np.uint64(12))
    return uint32_to_float_rz(u) * np.float32(2.0 ** -32)


def pr_fields(seed, n, frame_index, rounds=ROUNDS):
    """Photoreceptor-noise normal inputs of every pixel (local quads): (u, angle, sin_or_cos) as in leak_fields."""
    i = np.arange(n, dtype=np.uint64)
    j = (i & np.uint64(3)).astype(np.int64)
    w = _words(seed, i >> np.uint64(2), frame_index, 2, TAG_PR, rounds)
    return u01_open(_pick(w, j, 0, 2)), TWO_PI_F32 * u01_half(_pick(w, j, 1, 3)), (j & 1)


def normals(u, angle, sc):
    """float64 Box-Muller of the restated inputs (the device evaluates the same formula with fast intrinsics)."""
    r = np.sqrt(-2.0 * np.log(u.astype(np.float64)))
    a = angle.astype(np.float64)
    return np.where(sc == 0, r * np.cos(a), r * np.sin(a))
