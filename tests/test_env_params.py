"""CPU: per-env CACC scenario parameters (ENV_CONFIG <key>_range / slowdown_prob).

* parsing: the draw ranges of every field, point ranges for the keys left out, and every refusal message -- of the
  Python parser, of the one-env paths and of nmarl_cacc_draw_par itself (its checks run before any launch);
* the NumPy restatement of nmarl_cacc_draw_par against the keying include/nmarl.h documents, word by word;
* a config without the keys builds exactly what it builds without this feature: no table, the config-only entry
  points, the same nmarl_cacc_cfg.
"""
import ctypes as C

import numpy as np
import pytest

from deeprl_network_b200 import _lib as L
from deeprl_network_b200 import utils as U
from deeprl_network_b200.envs import cacc_env as CE
from env_par_ref import FIELDS, PAR_STREAM, draw_par
from helpers import load_cfg
from philox_ref import philox4x32_10, u01_from_bits

OPEN = dict(headway_target_range='15, 25', speed_target_range='12, 18', headway_st_range='3, 7',
            headway_go_range='30, 40', speed_max_range='25, 35', accel_min_range='-3, -2',
            accel_max_range='2, 3', slowdown_prob='0.5')


def _cfg(**over):
    return load_cfg('config_ma2c_nc_catchup.ini', **over)['ENV_CONFIG']


@pytest.fixture
def host_env(monkeypatch):
    """CACCEnv on CPU tensors: everything up to the first kernel launch runs without a GPU."""
    monkeypatch.setattr(L, 'require_cuda', lambda: None)
    return lambda cfg, n_env=None: CE.CACCEnv(cfg, n_env=n_env, device='cpu')


def test_parse_every_range_and_the_scenario_mix():
    sp = CE.parse_env_par(_cfg(**OPEN))
    assert sp['slowdown_prob'] == 0.5
    assert sp['ranges'] == dict(h_star=(15, 25), v_star=(12, 18), h_s=(3, 7), h_g=(30, 40), v_max=(25, 35),
                                u_min=(-3, -2), u_max=(2, 3))
    assert list(sp['ranges']) == list(L.ENV_PAR_FIELDS) == list(FIELDS)


def test_keys_left_out_are_point_ranges_at_the_nominal_value():
    sp = CE.parse_env_par(_cfg(speed_target_range='10, 20'))
    assert sp['slowdown_prob'] is None
    assert sp['ranges']['v_star'] == (10, 20)
    assert sp['ranges']['h_star'] == (20, 20) and sp['ranges']['h_s'] == (5, 5) and sp['ranges']['u_min'] == (-2.5, -2.5)
    assert CE.parse_env_par(_cfg(slowdown_prob='1'))['ranges']['h_g'] == (35, 35)


@pytest.mark.parametrize('over, msg', [
    (dict(speed_target_range='10'), 'speed_target_range = \'10\': expected two numbers "lo, hi"'),
    (dict(speed_target_range='10, 12, 14'), 'expected two numbers'),
    (dict(speed_max_range='a, b'), 'expected two numbers'),
    (dict(headway_target_range='25, 15'), 'headway_target_range = \'25, 15\': needs lo <= hi'),
    (dict(headway_st_range='1, 6'), 'headway_st (from 1) must exceed headway_min (1) for every draw'),
    (dict(headway_st='0.5', slowdown_prob='0'), 'headway_st (from 0.5) must exceed headway_min (1)'),
    (dict(headway_st_range='3, 36'), 'headway_st (up to 36) must stay below headway_go (from 35) for every draw'),
    (dict(headway_go_range='6, 40', headway_st_range='3, 7'), 'must stay below headway_go (from 6)'),
    (dict(accel_min_range='-3, 0'), 'accel_min (up to 0) must be negative for every draw'),
    (dict(accel_max_range='0, 2'), 'accel_max (from 0) must be positive for every draw'),
    (dict(speed_target_range='0, 15'), 'speed_target (from 0) must be positive for every draw'),
    (dict(headway_target_range='-1, 20'), 'headway_target (from -1) must be positive for every draw'),
    (dict(slowdown_prob='1.5'), 'ENV_CONFIG.slowdown_prob = 1.5: needs 0 <= p <= 1'),
    (dict(slowdown_prob='-0.1'), 'needs 0 <= p <= 1'),
])
def test_refusals(over, msg):
    with pytest.raises(ValueError) as e:
        CE.parse_env_par(_cfg(**over))
    assert msg in str(e.value)


@pytest.mark.parametrize('key', ['speed_target_range', 'slowdown_prob'])
def test_one_env_refuses_the_keys(host_env, key):
    val = '10, 20' if key.endswith('_range') else '0.5'
    with pytest.raises(ValueError) as e:
        host_env(_cfg(**{key: val}))                               # n_env = 1 from the config
    assert 'need batched training' in str(e.value) and key in str(e.value)
    with pytest.raises(ValueError, match='need batched training'):
        host_env(_cfg(n_env=8, **{key: val}), n_env=1)              # n_env = 1 from the constructor


def test_one_env_trainer_refuses_a_table(host_env):
    env = host_env(_cfg(n_env=4, **OPEN))

    class _Model:
        n_step = 60
    with pytest.raises(ValueError, match='batched training'):
        U.Trainer(env, _Model(), U.Counter(10, 10, 10), None)


def test_table_and_ranges_of_a_batched_env(host_env):
    env = host_env(_cfg(n_env=5, **OPEN))
    assert tuple(env.env_par.shape) == (5, 8) and C.sizeof(L.CaccEnvPar) == 64
    r = env._par_ranges
    assert list(r.lo) == [15, 12, 3, 30, 25, -3, 2] and list(r.hi) == [25, 18, 7, 40, 35, -2, 3]
    assert r.slowdown_prob == 0.5
    assert host_env(_cfg(n_env=5, speed_target_range='15, 15'))._par_ranges.slowdown_prob == -1.0   # scenario: config's


def test_config_without_keys_builds_what_it_built(host_env):
    """No key: no table, the nmarl_cacc_cfg of the config, and the evaluation config is the config itself."""
    for ini in ('config_ma2c_nc_catchup.ini', 'config_ia2c_slowdown.ini', 'config_ma2c_nc_grid5x5_stub.ini'):
        sec = load_cfg(ini, n_env=3)['ENV_CONFIG']
        assert CE.parse_env_par(sec) is None and CE.env_par_keys(sec) == []
        env = host_env(sec)
        assert env.env_par is None and env.par_spec is None and not hasattr(env, '_par_ranges')
        c = env.cfg
        assert (c.h_star, c.v_star, c.h_s, c.h_g, c.v_max, c.u_min, c.u_max) == \
            tuple(sec.getfloat(k) for k in CE.PAR_KEYS)
        assert c.scenario == (L.CATCHUP if 'catchup' in sec['scenario'] else L.SLOWDOWN)
        assert dict(CE.nominal_config(sec)) == dict(sec)


def test_nominal_config_drops_only_the_keys():
    sec = _cfg(n_env=64, **OPEN)
    nom = CE.nominal_config(sec)
    assert set(sec) - set(nom) == set(OPEN) and all(nom[k] == sec[k] for k in nom)
    assert CE.parse_env_par(nom) is None


def test_ctypes_mirrors_match_the_library():
    lib = L.lib()
    assert lib.nmarl_version() >= 107
    assert lib.nmarl_sizeof_cacc_env_par() == C.sizeof(L.CaccEnvPar) == 64
    assert lib.nmarl_sizeof_cacc_par_ranges() == C.sizeof(L.CaccParRanges) == 15 * 8
    assert lib.nmarl_sizeof_cacc_cfg() == C.sizeof(L.CaccCfg)


def _c_ranges(**over):
    r = L.CaccParRanges()
    lo = dict(h_star=15, v_star=12, h_s=3, h_g=30, v_max=25, u_min=-3, u_max=2)
    hi = dict(h_star=25, v_star=18, h_s=7, h_g=40, v_max=35, u_min=-2, u_max=3)
    for k, v in over.items():
        if k != 'p':
            (lo if k.endswith('_lo') else hi)[k[:-3]] = v
    for k, f in enumerate(L.ENV_PAR_FIELDS):
        r.lo[k], r.hi[k] = lo[f], hi[f]
    r.slowdown_prob = over.get('p', 0.5)
    return r


@pytest.mark.parametrize('over, msg', [
    (dict(v_max_lo=40), 'v_max range [40, 35] needs lo <= hi'),
    (dict(h_s_lo=1), 'needs h_min < h_s'),
    (dict(h_s_hi=31), 'needs h_s < h_g for every draw'),
    (dict(u_min_hi=0.5), 'needs u_min < 0'),
    (dict(u_max_lo=0), 'needs u_max > 0'),
    (dict(v_star_lo=0), 'needs v_star > 0'),
    (dict(h_star_lo=-2), 'needs h_star > 0'),
    (dict(p=1.5), 'slowdown_prob 1.5 > 1'),
])
def test_draw_par_checks_before_any_launch(over, msg):
    lib = L.lib()
    env_cfg = L.CaccCfg()
    env_cfg.h_min = 1.0
    dummy = 16                       # never dereferenced: the checks fail first
    rc = lib.nmarl_cacc_draw_par(C.byref(env_cfg), C.byref(_c_ranges(**over)), 4, 7, None, None, dummy, None)
    assert rc != 0 and msg in lib.nmarl_last_error().decode()


def test_draw_restatement_follows_the_documented_keying():
    """Lanes checked one by one: counter words (episode << 8 | k low, high), lane = env, tag 0x454E5650, key = seed;
    u from output words 0 and 1; value lo + u (hi - lo); scenario slow-down iff the k = 7 uniform < p."""
    seed = 0x1234_5678_9ABC_DEF0
    ranges = dict(zip(FIELDS, [(15, 25), (12, 18), (3, 7), (30, 40), (25, 35), (-3, -2), (2, 3)]))
    episode = np.array([0, 1, 7, 0x00FF_FFFF, 3], dtype=np.int64)
    tab = draw_par(seed, episode, ranges, 0.5, 0)
    for b in (0, 2, 3, 4):
        for k in range(8):
            c = (int(episode[b]) << 8) | k
            w = philox4x32_10((c & 0xFFFFFFFF, c >> 32, b, 0x454E5650), (seed & 0xFFFFFFFF, seed >> 32))
            u = ((int(w[0]) >> 5) * 2 ** 26 + (int(w[1]) >> 6)) / 2 ** 53
            assert u == float(u01_from_bits(w[0], w[1]))
            if k < 7:
                lo, hi = ranges[FIELDS[k]]
                assert tab[FIELDS[k]][b] == lo + u * (hi - lo)
            else:
                assert tab['scenario'][b] == (1 if u < 0.5 else 0)
    assert PAR_STREAM == 0x454E5650
    # point ranges give the value exactly; no slowdown_prob keeps the config's scenario
    pt = draw_par(seed, episode, {f: (r[0], r[0]) for f, r in ranges.items()}, None, 1)
    assert all(np.all(pt[f] == ranges[f][0]) for f in FIELDS) and np.all(pt['scenario'] == 1)
    assert np.all(draw_par(seed, episode, ranges, 0.0, 1)['scenario'] == 0)
    assert np.all(draw_par(seed, episode, ranges, 1.0, 0)['scenario'] == 1)


def test_draw_statistics():
    """Sanity of the whole table: every value inside its range, about the asked share of slow-down envs, and an env's
    next episode draws other values."""
    ranges = dict(zip(FIELDS, [(15, 25), (12, 18), (3, 7), (30, 40), (25, 35), (-3, -2), (2, 3)]))
    B = 4096
    a = draw_par(12, np.zeros(B), ranges, 0.3, 0)
    b = draw_par(12, np.ones(B), ranges, 0.3, 0)
    for f in FIELDS:
        lo, hi = ranges[f]
        assert np.all((a[f] >= lo) & (a[f] < hi)) and abs(a[f].mean() - (lo + hi) / 2) < 0.05 * (hi - lo)
        assert np.all(a[f] != b[f])
    assert abs(a['scenario'].mean() - 0.3) < 0.03
