"""CPU: the host restatement of the device random stream (tests/philox_ref.py) is Philox4x32-10, and the way the
kernels key it gives independent uniforms along every axis a rollout uses.  tests/test_gpu_philox.py then holds the
kernels to this restatement draw by draw."""
import numpy as np

import philox_ref as P


def _words(s):
    return [int(w, 16) for w in s.split()]


def test_known_answer_vectors():
    """Random123's published Philox4x32-10 vectors (kat_vectors: counter words, key words -> output words)."""
    kat = [('00000000 00000000 00000000 00000000', '00000000 00000000', '6627e8d5 e169c58d bc57ac4c 9b00dbd8'),
           ('ffffffff ffffffff ffffffff ffffffff', 'ffffffff ffffffff', '408f276d 41c83b0e a20bc7c6 6d5451fd'),
           ('243f6a88 85a308d3 13198a2e 03707344', 'a4093822 299f31d0', 'd16cfe09 94fdcceb 5001e420 24126ea1')]
    for ctr, key, out in kat:
        got = [int(x) for x in P.philox4x32_10(_words(ctr), _words(key))]
        assert got == _words(out), (ctr, key, ['%08x' % g for g in got])
    # vectorised over lanes: the three vectors in one call
    c = np.array([_words(k[0]) for k in kat], dtype=np.uint64).T
    k = np.array([_words(k[1]) for k in kat], dtype=np.uint64).T
    got = np.stack(P.philox4x32_10(c, k), axis=1)
    np.testing.assert_array_equal(got, np.array([_words(k[2]) for k in kat], dtype=np.uint32))


def test_u01_is_numpys_53_bit_recipe():
    assert P.u01_from_bits(0, 0) == 0.0
    assert P.u01_from_bits(0xFFFFFFFF, 0xFFFFFFFF) == 1.0 - 2.0 ** -53
    assert P.u01_from_bits(1 << 5, 0) == 2.0 ** -27 and P.u01_from_bits(0, 1 << 6) == 2.0 ** -53
    assert P.u01_from_bits(31, 63) == 0.0                   # the low 5 / 6 bits are dropped


def _lag1(x, axis):
    a = np.moveaxis(x, axis, 0)
    return float(np.corrcoef(a[:-1].ravel(), a[1:].ravel())[0, 1]), a[:-1].size


def test_action_stream_is_uniform_and_uncorrelated_along_every_axis():
    """2^20 draws laid out [counter t][agent][env] as a rollout keys them: lane = agent * B + env, counter = t."""
    seed, T, N, B = 0x1234567890ABCDEF, 16, 8, 8192
    u = np.stack([P.action_uniforms(seed, t, N, B) for t in range(T)])
    assert u.shape == (T, N, B) and u.min() >= 0.0 and u.max() < 1.0
    n = u.size
    counts = np.bincount((u.ravel() * 64).astype(int), minlength=64)
    chi2 = float(((counts - n / 64) ** 2 / (n / 64)).sum())
    assert chi2 < 63 + 4 * np.sqrt(2 * 63), chi2            # 63 degrees of freedom: mean 63, sd sqrt(126)
    for axis in range(3):
        r, m = _lag1(u, axis)
        assert abs(r) < 4 / np.sqrt(m), ('lag-1 correlation along axis %d' % axis, r)
    assert len(np.unique(u)) == n                           # no draw is shared between steps, agents or envs
    # the high counter word and both key words reach the output
    base = P.action_uniforms(seed, 5, N, 64)
    assert not np.array_equal(base, P.action_uniforms(seed, 5 + 2 ** 32, N, 64))
    assert not np.array_equal(base, P.action_uniforms(seed ^ 1, 5, N, 64))
    assert not np.array_equal(base, P.action_uniforms(seed ^ (1 << 32), 5, N, 64))


def test_reset_stream_is_independent_of_the_action_stream():
    """Env resets (lane = env, counter = episode << 8 | platoon) share seed, counter and lane values with the action
    stream; the stream tag alone must make them unrelated."""
    seed, E, Pn, B = 12, 8, 5, 4096
    r = np.stack([P.reset_uniforms(seed, np.full(B, ep), Pn, B) for ep in range(E)])          # [E, P, B]
    a = np.stack([[P.philox_u01(seed, (ep << 8) | p, np.arange(B), P.ACTION_STREAM) for p in range(Pn)] for ep in range(E)])
    assert r.shape == a.shape == (E, Pn, B)
    n = r.size
    assert abs(float(np.corrcoef(r.ravel(), a.ravel())[0, 1])) < 4 / np.sqrt(n)
    assert not np.any(r == a)
    for axis in range(3):                                   # episodes, platoons and envs draw independently
        c, m = _lag1(r, axis)
        assert abs(c) < 4 / np.sqrt(m), (axis, c)
    counts = np.bincount((r.ravel() * 64).astype(int), minlength=64)
    assert float(((counts - n / 64) ** 2 / (n / 64)).sum()) < 63 + 4 * np.sqrt(2 * 63)


def test_inverse_cdf_rules():
    pi = np.array([[0.25, 0.25, 0.5], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]], dtype=np.float32)
    for scaled in (False, True):
        np.testing.assert_array_equal(P.inverse_cdf(pi, [0.0, 0.999, 0.0], scaled), [0, 0, 2])
        np.testing.assert_array_equal(P.inverse_cdf(pi, [0.25, 0.5, 0.7], scaled), [1, 0, 2])      # cdf <= u: 'right'
        np.testing.assert_array_equal(P.inverse_cdf(pi[:1], [0.4999], scaled), [1])
        assert P.inverse_cdf(np.ones((1, 1), np.float32), [0.3], scaled)[0] == 0                    # n_a = 1
