"""GPU: per-env CACC scenario parameters (nmarl_cacc_draw_par, nmarl_cacc_reset_pe, nmarl_cacc_step_pe, VecTrainer).

Env b of a batch must behave exactly like the reference CACCEnv constructed with env b's parameter values:
* the device draw equals its NumPy restatement (tests/env_par_ref.py) bit for bit, for a partial mask and several
  episode counters;
* B envs with every range open and mixed scenarios, the reset and 600 random-action steps, against the float64 oracle
  env built from each env's drawn row -- 257 envs of an 8-vehicle chain, 40 of a 5x5 grid of platoons and 8 of a
  128-vehicle chain (the scalar oracle steps ~0.4 ms per 8-vehicle env).  Tolerances are those of tests/test_gpu_env.py (CUDA's and glibc's float64 cos() may differ by an ulp);
* point ranges at the nominal values give the config-only kernels' outputs bit for bit;
* an env that resets draws fresh parameters and the others keep theirs;
* VecTrainer: graph replay == eager, run-to-run determinism, env_par.csv, nominal greedy tests; main.py train +
  evaluate.
"""
import configparser
import os

import numpy as np
import pytest
import torch

import main
from deeprl_network_b200 import utils as U
from env_par_ref import FIELDS, draw_par, oracle_env, row
from helpers import ROOT, load_cfg
from philox_ref import reset_uniforms

pytestmark = pytest.mark.gpu

OPEN = dict(headway_target_range='15, 25', speed_target_range='12, 18', headway_st_range='3, 7',
            headway_go_range='30, 40', speed_max_range='25, 35', accel_min_range='-3, -2',
            accel_max_range='2, 3', slowdown_prob='0.5')
RANGES = dict(zip(FIELDS, [(15, 25), (12, 18), (3, 7), (30, 40), (25, 35), (-3, -2), (2, 3)]))


def _env(ini='config_ma2c_nc_catchup.ini', B=257, **over):
    from deeprl_network_b200.envs.cacc_env import CACCEnv
    cp = load_cfg(ini, n_env=B, **over)
    return cp, CACCEnv(cp['ENV_CONFIG'])


def test_draw_equals_numpy_restatement():
    cp, env = _env(**OPEN)
    B = env.n_env
    rs = np.random.RandomState(0)
    seed = 0xDEADBEEF12345
    for it in range(4):
        ep = rs.randint(0, [1, 5, 1000, 2 ** 24][it], size=B).astype(np.int32)
        env.episode_dev.copy_(torch.as_tensor(ep))
        mask = (rs.rand(B) < 0.6).astype(np.float32)
        env.env_par.fill_(-7.0)
        before = env.par_table()
        env.reset_device(u01=None, mask=torch.as_tensor(mask).cuda(), philox_seed=seed)
        got = env.par_table()
        want = draw_par(seed, ep, RANGES, 0.5, 0)
        m = mask != 0
        for k in FIELDS + ('scenario',):
            np.testing.assert_array_equal(got[k][m], want[k][m], err_msg=k)
            np.testing.assert_array_equal(got[k][~m], before[k][~m], err_msg=k)
        np.testing.assert_array_equal(env.episode_dev.cpu().numpy(), ep + m)     # the reset moved the counters
        assert 0 < got['scenario'][m].sum() < m.sum()


def _run_vs_oracle(ini, B, steps, seed, **over):
    """Reset (Philox uniforms) + `steps` random-action steps of B envs against per-env, per-platoon oracles."""
    cp, env = _env(ini, B, **OPEN, **over)
    N, Lp = env.n_agent, env.platoon_len
    P = N // Lp
    env.reset_device(u01=None, philox_seed=seed)
    tab = draw_par(seed, np.zeros(B), RANGES, 0.5, 0)
    got = env.par_table()
    for k in FIELDS + ('scenario',):
        np.testing.assert_array_equal(got[k], tab[k], err_msg=k)
    assert 0 < tab['scenario'].sum() < B
    u = reset_uniforms(seed, np.zeros(B), P, B)
    sub = load_cfg(ini, n_vehicle=Lp, **{k: v for k, v in over.items() if k != 'n_vehicle'})['ENV_CONFIG']
    orc = [[oracle_env(sub, row(tab, b)) for _ in range(P)] for b in range(B)]
    for b in range(B):
        for p in range(P):
            orc[b][p].reset(u01=u[p, b])
    h0 = np.stack([np.concatenate([o.hs_cur for o in orc[b]]) for b in range(B)], 1)
    v0 = np.stack([np.concatenate([o.vs_cur for o in orc[b]]) for b in range(B)], 1)
    np.testing.assert_array_equal(env.hs.cpu().numpy(), h0)
    np.testing.assert_array_equal(env.vs.cpu().numpy(), v0)
    rs = np.random.RandomState(seed)
    acts = rs.randint(0, 4, size=(steps, N, B)).astype(np.int32)
    acts[:, :, 1:17] = 0              # no acceleration command: the slow-down platoons among these collide
    alive = np.ones(B, bool)
    n_done = np.zeros(steps, int)
    for t in range(steps):
        env.step_device(torch.as_tensor(acts[t]).cuda())
        hs, vs, us = (x.cpu().numpy() for x in (env.hs, env.vs, env.us))
        obs = env.obs_dev[..., :5].cpu().numpy()
        rew, grew = env.reward_dev.cpu().numpy(), env.greward_dev.cpu().numpy()
        done, col = env.done_dev.cpu().numpy() != 0, env.collision_dev.cpu().numpy() != 0
        if P > 1:
            alive &= ~col                         # the platoons of a grid env share one collision latch: stop there
        live = np.nonzero(alive)[0]
        o_h, o_v, o_u = (np.empty((N, len(live))) for _ in range(3))
        o_obs = np.empty((N, len(live), 5))
        o_r, o_g, o_d, o_c = np.empty((rew.shape[0], len(live))), np.empty(len(live)), [], []
        for j, b in enumerate(live):
            outs = [orc[b][p].step(acts[t, p * Lp:(p + 1) * Lp, b]) for p in range(P)]
            o_h[:, j] = np.concatenate([o.hs_cur for o in orc[b]])
            o_v[:, j] = np.concatenate([o.vs_cur for o in orc[b]])
            o_u[:, j] = np.concatenate([o.us_cur for o in orc[b]])
            o_obs[:, j] = np.concatenate([np.stack([x[:5] for x in out[0]]) for out in outs])
            if P == 1:
                _, r, d, gr = outs[0]
                o_r[:, j], o_g[j] = r, gr
                o_d.append(d)
                o_c.append(orc[b][0].collision)
        np.testing.assert_allclose(hs[:, live], o_h, rtol=1e-11, atol=1e-11, err_msg='h, step %d' % t)
        np.testing.assert_allclose(vs[:, live], o_v, rtol=1e-11, atol=1e-11, err_msg='v, step %d' % t)
        np.testing.assert_allclose(us[:, live], o_u, rtol=1e-9, atol=1e-9, err_msg='u, step %d' % t)
        np.testing.assert_allclose(obs[:, live], o_obs.astype(np.float32), rtol=0, atol=1e-6, err_msg='obs %d' % t)
        if P == 1:
            np.testing.assert_array_equal(done[live], o_d, err_msg='done, step %d' % t)
            np.testing.assert_array_equal(col[live], o_c, err_msg='collision, step %d' % t)
            np.testing.assert_allclose(grew[live], o_g, rtol=1e-9, atol=1e-9, err_msg='global reward, step %d' % t)
            np.testing.assert_allclose(rew[:, live], o_r, rtol=1e-9, atol=1e-9, err_msg='reward, step %d' % t)
            alive &= ~done
        n_done[t] = done.sum()
    return env, alive, n_done


def test_every_env_matches_its_oracle_chain():
    env, alive, n_done = _run_vs_oracle('config_ma2c_nc_catchup.ini', 257, 600, 12)
    assert alive.sum() == 0 and n_done[-1] == 257              # every episode ended, at T at the latest
    assert n_done[:-1].sum() > 0                               # and some at an earlier collision boundary
    assert np.all(env.t_dev.cpu().numpy() == 600)


def test_every_env_matches_its_oracle_grid():
    env, alive, _ = _run_vs_oracle('config_ma2c_nc_grid5x5_stub.ini', 40, 600, 5)
    assert env.n_agent == 25 and env.platoon_len == 5


def test_every_env_matches_its_oracle_128_chain():
    env, alive, n_done = _run_vs_oracle('config_ma2c_nc_slowdown.ini', 8, 600, 9, n_vehicle=128)
    assert env.n_agent == 128 and n_done[-1] == 8


@pytest.mark.parametrize('ini, p', [('config_ma2c_nc_catchup.ini', 0), ('config_ma2c_nc_slowdown.ini', 1),
                                    ('config_ia2c_slowdown.ini', 1), ('config_ma2c_nc_grid5x5_stub.ini', 0)])
def test_point_ranges_are_bit_identical_to_the_config_kernels(ini, p):
    sec = load_cfg(ini)['ENV_CONFIG']
    keys = {k + '_range': '%s, %s' % (sec[k], sec[k]) for k in ('headway_target', 'speed_target', 'headway_st',
                                                             'headway_go', 'speed_max', 'accel_min', 'accel_max')}
    B = 129
    _, ref = _env(ini, B)
    _, pe = _env(ini, B, slowdown_prob=p, **keys)
    assert ref.env_par is None and pe.env_par is not None
    rs = np.random.RandomState(1)
    state = lambda e: [e.hs, e.vs, e.us, e.v_init, e.t_dev, e.collision_dev, e.obs_dev, e.fp_dev, e.reward_dev,
                       e.greward_dev, e.done_dev, e.episode_dev]
    for e in (ref, pe):
        e.reset_device(u01=None, philox_seed=77)
    for t in range(600):
        a = torch.as_tensor(rs.randint(0, 4, size=(ref.n_agent, B)).astype(np.int32)).cuda()
        for e in (ref, pe):
            e.train_mode = t < 400
            e.step_device(a)
        if t == 300:                                        # a masked reset in the middle
            m = torch.as_tensor((rs.rand(B) < 0.5).astype(np.float32)).cuda()
            for e in (ref, pe):
                e.reset_device(u01=None, mask=m, philox_seed=77)
        for x, y in zip(state(ref), state(pe)):
            assert torch.equal(x, y), t


def test_resets_redraw_only_the_envs_that_reset():
    cp, env = _env(B=64, **OPEN)
    seed, B = 31, 64
    env.reset_device(u01=None, philox_seed=seed)
    rs = np.random.RandomState(2)
    ep = np.zeros(B, np.int64)
    tab = env.par_table()
    for boundary in range(4):
        acts = rs.randint(0, 4, size=(60, env.n_agent, B)).astype(np.int32)
        acts[:, :, :16] = 0                                 # no acceleration command: slow-down platoons collide
        for t in range(60):
            env.step_device(torch.as_tensor(acts[t]).cuda())
        # envs whose episode ended (collision at this batch boundary), plus a staggered subset, start a new one
        done = (env.done_dev.cpu().numpy() != 0) | (rs.rand(B) < 0.25)
        assert 0 < done.sum() < B, boundary
        env.reset_device(u01=None, mask=torch.as_tensor(done.astype(np.float32)).cuda(), philox_seed=seed)
        ep += done
        new = env.par_table()
        want = draw_par(seed, ep, RANGES, 0.5, 0)
        for k in FIELDS:
            np.testing.assert_array_equal(new[k][done], want[k][done])
            assert np.all(new[k][done] != tab[k][done])      # fresh values for a new episode
            np.testing.assert_array_equal(new[k][~done], tab[k][~done])
        np.testing.assert_array_equal(new['scenario'][~done], tab['scenario'][~done])
        np.testing.assert_array_equal(env.episode_dev.cpu().numpy(), ep + 1)
        tab = new


# ---- VecTrainer ------------------------------------------------------------------------------------------------------
def _trainer(graph, B=256, **over):
    from deeprl_network_b200.agents.models import MA2C_NC
    cp, env = _env('config_ma2c_nc_catchup.ini', B, **OPEN, **over)
    model = MA2C_NC(env.n_s_ls, env.n_a_ls, env.neighbor_mask, env.distance_mask, env.coop_gamma, 10 ** 6,
                    cp['MODEL_CONFIG'], seed=12, n_env=B)
    return cp, env, model, U.VecTrainer(env, model, graph=graph)


def _three_updates(graph):
    cp, env, model, vt = _trainer(graph)
    assert model.engine.use_tc
    vt.start()
    tabs = []
    for k in range(3):
        vt.update()
        vt.log_rewards(k)
        tabs.append(env.env_par.clone())
    torch.cuda.synchronize()
    model.engine.check_tc()
    e = model.engine
    return dict(params=e.params.clone(), grew=e.grew_buf.clone(), t=env.t_dev.clone(), hs=env.hs.clone(),
                episode=env.episode_dev.clone(), par=torch.stack(tabs)), vt


def test_vec_trainer_graph_equals_eager_and_is_deterministic(tmp_path):
    eager, _ = _three_updates(False)
    graph, vt = _three_updates(True)
    again, _ = _three_updates(True)
    for k in eager:
        assert torch.equal(eager[k], graph[k]), k
        assert torch.equal(graph[k], again[k]), k
    vt.write_csv(str(tmp_path) + '/')
    import pandas as pd
    df = pd.read_csv(tmp_path / 'env_par.csv')
    assert len(df) == 3 and list(df['step']) == [0, 1, 2]
    for f in FIELDS:
        lo, hi = RANGES[f]
        assert np.all(df[f + '_min'] >= lo) and np.all(df[f + '_max'] < hi)
        assert np.all(df[f + '_min'] <= df[f + '_mean']) and np.all(df[f + '_mean'] <= df[f + '_max'])
    assert np.all((df['slowdown_mean'] > 0.3) & (df['slowdown_mean'] < 0.7))
    assert list(pd.read_csv(tmp_path / 'train_reward.csv').columns)[1:] == ['agent', 'step', 'test_id',
                                                                           'avg_reward', 'std_reward']


def test_greedy_tests_use_the_nominal_values():
    """BatchedEvaluator built from a config with the keys == one built from the config without them, same weights."""
    _, env, model, vt = _trainer(False, B=128, test_seeds='2000,2010,2020')
    vt.start()
    vt.update()
    seeds = env.test_seeds
    with_keys = load_cfg('config_ma2c_nc_catchup.ini', n_env=128, test_seeds='2000,2010,2020', **OPEN)['ENV_CONFIG']
    plain = load_cfg('config_ma2c_nc_catchup.ini', n_env=128, test_seeds='2000,2010,2020')['ENV_CONFIG']
    a = U.BatchedEvaluator(with_keys, model).test_rewards(seeds)
    b = U.BatchedEvaluator(plain, model).test_rewards(seeds)
    assert a == b


def test_cli_train_then_evaluate(tmp_path):
    cp = configparser.ConfigParser()
    cp.read(os.path.join(ROOT, 'config', 'config_ma2c_nc_catchup.ini'))
    n_env = 128
    cp['ENV_CONFIG'].update(dict(n_env=str(n_env), **OPEN))
    cp['TRAIN_CONFIG'].update(dict(total_step=str(2 * 60 * n_env), log_interval=str(60 * n_env)))
    ini = str(tmp_path / 'exp.ini')
    with open(ini, 'w') as f:
        cp.write(f)
    base = str(tmp_path / 'run')
    main.train(main.parse_args(['--base-dir', base, 'train', '--config-dir', ini]))
    assert sorted(os.listdir(base + '/data')) == ['env_par.csv', 'exp.ini', 'train_reward.csv']
    import pandas as pd
    assert len(pd.read_csv(base + '/data/env_par.csv')) == len(pd.read_csv(base + '/data/train_reward.csv')) == 2
    main.evaluate(main.parse_args(['--base-dir', base, 'evaluate', '--evaluation-seeds', '2000,2010']))
    out = sorted(os.listdir(base + '/eva_data'))
    assert out == ['catchup_ma2c_nc_control.csv', 'catchup_ma2c_nc_traffic.csv']
    # one-env training refuses the keys, naming batched training
    cp['ENV_CONFIG']['n_env'] = '1'
    with open(ini, 'w') as f:
        cp.write(f)
    with pytest.raises(ValueError, match='batched training'):
        main.train(main.parse_args(['--base-dir', str(tmp_path / 'one'), 'train', '--config-dir', ini]))
