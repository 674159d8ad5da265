"""A numpy restatement of the device draws of b2second.augment.DeviceDrawer (csrc/augment_draws.cu), from the
generator contract in INTEGRATION.md: Philox4x64-10 keyed by (seed, step) at counter (frame, stream, index, 0), numpy's
53-bit uniforms, Box-Muller normals, and a keyed Feistel permutation with cycle walking for the shuffle.

Everything is vectorised over uint64 arrays; the 64 x 64 -> 128-bit products are built from 32-bit limbs, so nothing
here uses numpy.random.Philox (the tests compare against it)."""
import math

import numpy as np

from b2second import augment

M0, M1 = np.uint64(0xD2E7470EE14C6C93), np.uint64(0xCA5A826395121157)     # Philox4x64 multipliers
W0, W1 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBB67AE8584CAA73B)     # its Weyl key increments
ROUNDS = 10
NUM_TRY = augment.NUM_TRY
TWO_PI = 2.0 * math.pi
S_LOC, S_ROT, S_FRAME, S_PERM = 0, 1, 2, 3                                # the counter's stream word

_M32 = np.uint64(0xFFFFFFFF)
_32 = np.uint64(32)


def _u64(v):
    return np.atleast_1d(np.asarray(v, dtype=np.uint64))


def _mulhilo(a, b):
    """(hi, lo) 64-bit words of the 128-bit product of uint64 arrays"""
    a0, a1, b0, b1 = a & _M32, a >> _32, b & _M32, b >> _32
    p00, p01, p10, p11 = a0 * b0, a0 * b1, a1 * b0, a1 * b1
    mid = (p00 >> _32) + (p01 & _M32) + (p10 & _M32)
    hi = p11 + (p01 >> _32) + (p10 >> _32) + (mid >> _32)
    return hi, a * b


def philox(key, counter):
    """Philox4x64-10 -> four uint64 arrays.  key = (k0, k1), counter = (c0, c1, c2, c3); each word broadcasts."""
    with np.errstate(over="ignore"):
        k0, k1 = (_u64(k) for k in key)
        c = np.broadcast_arrays(*[_u64(w) for w in counter], k0, k1)
        c0, c1, c2, c3, k0, k1 = (np.array(w) for w in c)
        for r in range(ROUNDS):
            if r:
                k0, k1 = k0 + W0, k1 + W1
            hi0, lo0 = _mulhilo(M0, c0)
            hi1, lo1 = _mulhilo(M1, c2)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
    return c0, c1, c2, c3


def uniform01(w):
    """numpy's double from a 64-bit word: (w >> 11) * 2**-53"""
    return (w >> np.uint64(11)).astype(np.float64) * (1.0 / 9007199254740992.0)


def uniform(w, lo, hi):
    return lo + (hi - lo) * uniform01(w)


def box_muller(wa, wb):
    """(r cos t, r sin t) with r = sqrt(-2 ln(1 - u(wa))), t = 2 pi u(wb), through libm"""
    r = np.sqrt(-2.0 * np.log(1.0 - uniform01(wa)))
    t = TWO_PI * uniform01(wb)
    return r * np.cos(t), r * np.sin(t)


def feistel_bits(n):
    """k: the smallest k >= 1 with 4**k >= n"""
    k = 1
    while 4 ** k < n:
        k += 1
    return k


def permutation(key, frame, n):
    """perm[i] = pi(i) for a frame of n points: 4 Feistel rounds on (L, R) of k bits each, cycle-walked into [0, n)"""
    if n <= 1:
        return np.arange(n, dtype=np.int32)
    k = feistel_bits(n)
    mask = np.uint64((1 << k) - 1)
    x = np.arange(n, dtype=np.uint64)
    todo = np.ones(n, dtype=bool)
    while todo.any():
        v = x[todo]
        L, R = v >> np.uint64(k), v & mask
        for r in range(4):
            f = philox(key, (frame, S_PERM, r, R))[0] & mask
            L, R = R, L ^ f
        x[todo] = (L << np.uint64(k)) | R
        todo = x >= np.uint64(n)
    return x.astype(np.int32)


def draws(settings, seed, step, num_gt, num_points, frame_base=0):
    """the draws DeviceDrawer.draw makes for frames frame_base + b with the given per-frame counts, as host arrays in
    augment.Draws' layout"""
    s = settings
    key = (seed, step)
    noise = augment.object_noise_enabled(s)
    std = [float(v) for v in s.groundtruth_localization_noise_std]
    rot = [float(v) for v in s.groundtruth_rotation_uniform_noise]
    tstd = [float(v) for v in s.global_translate_noise_std]
    translate = not all(e == 0 for e in tstd)
    locs, rots, frames, perms = [], [], [], []
    for b, (n, npts) in enumerate(zip(num_gt, num_points)):
        f = frame_base + b
        if noise:
            idx = np.arange(n * NUM_TRY, dtype=np.uint64)
            w = philox(key, (f, S_LOC, idx, 0))
            n0, n1 = box_muller(w[0], w[1])
            n2 = box_muller(w[2], w[3])[0]
            locs.append(np.stack([n0 * std[0], n1 * std[1], n2 * std[2]], -1).reshape(n, NUM_TRY, 3))
            rots.append(uniform(philox(key, (f, S_ROT, idx, 0))[0], rot[0], rot[1]).reshape(n, NUM_TRY))
        w = philox(key, (f, S_FRAME, 0, 0))
        flip_x, flip_y = uniform01(w[0])[0] < 0.5, uniform01(w[1])[0] < 0.5
        angle = uniform(w[2], *s.global_rotation_uniform_noise)[0]
        scale = uniform(w[3], *s.global_scaling_uniform_noise)[0]
        t = [0.0, 0.0, 0.0]
        if translate:
            w = philox(key, (f, S_FRAME, 1, 0))
            n0, n1 = box_muller(w[0], w[1])
            n2 = box_muller(w[2], w[3])[0]
            t = [n0[0] * tstd[0], n1[0] * tstd[1], n2[0] * tstd[0]]
        frames.append([float(bool(flip_y) and s.random_flip_y), float(bool(flip_x) and s.random_flip_x),
                       float(translate), angle, scale, *t])
        if s.shuffle_points:
            perms.append(permutation(key, f, int(npts)))
    return augment.Draws(
        loc_noise=(np.concatenate(locs) if locs else np.zeros((0, NUM_TRY, 3))) if noise else None,
        rot_noise=(np.concatenate(rots) if rots else np.zeros((0, NUM_TRY))) if noise else None,
        frame=np.array(frames, np.float64).reshape(-1, 8),
        perm=(np.concatenate(perms) if perms else np.zeros(0, np.int32)) if s.shuffle_points else None,
        num_gt=[int(v) for v in num_gt], num_points=[int(v) for v in num_points])
