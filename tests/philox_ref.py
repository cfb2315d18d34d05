"""NumPy restatement of the device random stream, written from the definition of Philox4x32-10 (Salmon, Moraes, Dror,
Shaw: "Parallel random numbers: as easy as 1, 2, 3", SC'11), not from csrc/common.cuh, so that a wrong constant or a
swapped word in the kernels shows up as a disagreement instead of being mirrored.

One Philox round on the counter (c0, c1, c2, c3) with the key (k0, k1):
    (h0, l0) = M0 * c0,  (h1, l1) = M1 * c2              (32 x 32 -> 64-bit products, high and low halves)
    (c0, c1, c2, c3) <- (h1 ^ c1 ^ k0,  l1,  h0 ^ c3 ^ k1,  l0)
and between rounds the key is bumped by the Weyl constants (k0, k1) += (W0, W1).  Philox4x32-10 is ten rounds.

How the kernels key it (include/nmarl.h): key = the 64-bit seed (low word first), counter words = (counter low,
counter high, lane, stream tag).  A uniform is NumPy's 53-bit random_sample recipe on output words 0 and 1.
"""
import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57          # multipliers
W0, W1 = 0x9E3779B9, 0xBB67AE85          # key schedule: golden ratio and sqrt(3) - 1
ACTION_STREAM = 0x41435431               # stream tag of action sampling: lane = agent * B + env, counter = p-call index
RESET_STREAM = 0x454E5601                # stream tag of env resets: lane = env, counter = episode << 8 | platoon
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: four uint32 words, key: two, each a scalar or an array (broadcast together) -> four uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & MASK32 for x in ctr]
    k = [np.asarray(x, dtype=np.uint64) & MASK32 for x in key]
    for rnd in range(10):
        if rnd:
            k = [(k[0] + np.uint64(W0)) & MASK32, (k[1] + np.uint64(W1)) & MASK32]
        p0, p1 = np.uint64(M0) * c[0], np.uint64(M1) * c[2]           # < 2^64: exact in uint64
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & MASK32, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & MASK32]
    return [x.astype(np.uint32) for x in np.broadcast_arrays(*c)]


def u01_from_bits(a, b):
    """NumPy's random_sample: 27 high bits of a and 26 high bits of b make a 53-bit fraction in [0, 1)."""
    a, b = np.asarray(a, dtype=np.uint32), np.asarray(b, dtype=np.uint32)
    return ((a >> np.uint32(5)).astype(np.float64) * 67108864.0 + (b >> np.uint32(6)).astype(np.float64)) / 9007199254740992.0


def philox_u01(seed, counter, lane, stream):
    """seed, counter: 64-bit integers (counter may be a uint64 array), lane: uint32 (array) -> float64 uniforms."""
    seed = int(seed) & (2 ** 64 - 1)
    counter = np.asarray(counter, dtype=np.uint64)
    out = philox4x32_10((counter & MASK32, counter >> np.uint64(32), lane, stream), (seed & 0xFFFFFFFF, seed >> 32))
    return u01_from_bits(out[0], out[1])


def action_uniforms(seed, counter, n_agent, B):
    """[n_agent, B] uniforms of the p-call with this counter (device counter + rng_offset, modulo 2^64)."""
    lane = np.arange(n_agent * B, dtype=np.uint64).reshape(n_agent, B)
    return philox_u01(seed, int(counter) & (2 ** 64 - 1), lane, ACTION_STREAM)


def reset_uniforms(seed, episode, n_platoon, B):
    """[n_platoon, B] uniforms of an env reset; episode: [B] resets each env has seen before this one."""
    episode = np.asarray(episode, dtype=np.uint64).reshape(1, B)
    counter = (episode << np.uint64(8)) | np.arange(n_platoon, dtype=np.uint64).reshape(n_platoon, 1)
    return philox_u01(seed, counter, np.arange(B, dtype=np.uint64).reshape(1, B), RESET_STREAM)


def inverse_cdf(pi, u, scaled):
    """The action a kernel draws from its own float32 pi [..., n_a] and the uniform u [...]: the cdf is built by
    sequential float64 adds in action order (s = its last entry), the action is the number of entries at or below u.
    FP32-FFMA kernel (scaled=False): cdf / s <= u, np.random.choice's rule.  Tensor-core kernel (scaled=True):
    cdf <= u * s, the same draw without the divisions.  Clipped to the last action."""
    pi = np.asarray(pi, dtype=np.float32).astype(np.float64)
    n_a = pi.shape[-1]
    cdf = np.empty_like(pi)
    s = np.zeros(pi.shape[:-1])
    for a in range(n_a):
        s = s + pi[..., a]
        cdf[..., a] = s
    u = np.asarray(u, dtype=np.float64)[..., None]
    below = (cdf <= u * s[..., None]) if scaled else (cdf / s[..., None] <= u)
    return np.minimum(below.sum(-1), n_a - 1).astype(np.int32)
