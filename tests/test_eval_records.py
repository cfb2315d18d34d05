"""CPU: the host half of batched evaluation.  Records of many episodes laid out as the device recorder leaves them
([T+1][E][N], garbage after each episode's end), split into passes and turned into the two CSV files, must equal
byte for byte what the one-env path writes while it steps: CACCEnv's per-step recording (the code Evaluator runs),
fed by the oracle env."""
import itertools
import logging

import numpy as np
import pytest

from deeprl_network_b200 import utils as U
from deeprl_network_b200.envs.cacc_env import CACCEnv
from helpers import load_cfg
from oracle.cacc import OracleCACC

SEEDS = [2000, 2010, 2020, 2030, 2040]


class _OneEnvRecorder:
    """The attributes CACCEnv's recording methods use, so that they run on the oracle env's states."""

    def __init__(self, name, agent, dt, output_path):
        self.name, self.agent, self.dt, self.output_path = name, agent, dt, output_path
        self.is_record, self.control_data, self.traffic_data = True, [], []


def _actions(k, T, N):
    """Episode k's joint actions: all 0 (followers keep their speed: the slow-down platoon collides), all 3, random."""
    if k % 3 == 0:
        return np.zeros((T, N), dtype=np.int32)
    if k % 3 == 1:
        return np.full((T, N), 3, dtype=np.int32)
    return np.random.RandomState(k).randint(0, 4, size=(T, N)).astype(np.int32)


def _run_oracle(cfg, out):
    """One-env path: returns the device-recorder layout of the same episodes and the expected log lines."""
    env = OracleCACC(cfg)
    env.init_test_seeds(SEEDS)
    env.train_mode = False
    T, N, E = env.T, env.n_agent, len(SEEDS)
    rec = _OneEnvRecorder(env.name, env.agent, env.dt, out)
    steps = np.zeros(E, dtype=np.int32)
    action = np.full((T + 1, E, N), 7, dtype=np.int32)                   # slots after an episode's end: garbage
    reward = np.full((T + 1, E), 1e9)
    hs, vs, us = (np.full((T + 1, E, N), np.nan) for _ in range(3))
    lines = []
    for k in range(E):
        env.reset(test_ind=k)
        rec.cur_episode, rec.t, rec.rewards = k + 1, 0, [0]
        rec._trace = [np.stack([env.hs_cur, env.vs_cur, env.us_cur])]
        action[0, k], reward[0, k] = 0, 0.0
        hs[0, k], vs[0, k], us[0, k] = env.hs_cur, env.vs_cur, env.us_cur
        acts = _actions(k, T, N)
        for t in range(T):
            _, _, done, g = env.step(acts[t])
            rec.t += 1
            rec.rewards.append(g)
            CACCEnv._log_control_data(rec, acts[t].astype(np.int64), g)
            rec._trace.append(np.stack([env.hs_cur, env.vs_cur, env.us_cur]))
            action[t + 1, k], reward[t + 1, k] = acts[t], g
            hs[t + 1, k], vs[t + 1, k], us[t + 1, k] = env.hs_cur, env.vs_cur, env.us_cur
            if done:
                CACCEnv._log_traffic_data(rec)
                break
        steps[k] = rec.t
        lines.append('test %i, avg reward %.2f' % (k, np.mean(np.array(rec.rewards[1:]))))
    CACCEnv.output_data(rec)
    return (steps, action, reward, hs, vs, us), lines, T


@pytest.mark.parametrize('cfg_name', ['config_ma2c_nc_catchup.ini', 'config_ma2c_cnet_slowdown.ini'])
def test_batched_records_match_one_env_recording(cfg_name, tmp_path, caplog):
    cfg = load_cfg(cfg_name)['ENV_CONFIG']
    one, many = tmp_path / 'one', tmp_path / 'many'
    one.mkdir(), many.mkdir()
    arrays, lines, T = _run_oracle(cfg, str(one) + '/')
    steps = arrays[0]
    if 'slowdown' in cfg_name:
        assert (steps < T).any(), 'no episode ended early'
    name, agent, dt = cfg['scenario'].split('_')[1], cfg['agent'], float(cfg['control_interval_sec'])
    files = sorted(p.name for p in one.iterdir())
    assert files == ['%s_%s_%s.csv' % (name, agent, k) for k in ('control', 'traffic')]
    for E in (len(SEEDS), 1, 2, 3):                       # passes of E envs; the last one may be shorter
        out = many / str(E)
        out.mkdir()
        caplog.clear()
        passes = [U.split_episodes(c0, *(a[c0:c0 + E] if a.ndim == 1 else a[:, c0:c0 + E] for a in arrays))
                  for c0 in range(0, len(SEEDS), E)]
        with caplog.at_level(logging.INFO):
            U.write_episode_records(itertools.chain(*passes), str(out) + '/', name, agent, dt)
        assert [r.getMessage() for r in caplog.records if r.getMessage().startswith('test ')] == lines
        for f in files:
            assert (out / f).read_bytes() == (one / f).read_bytes(), (E, f)


def test_no_output_path_writes_nothing(tmp_path, caplog):
    cfg = load_cfg('config_ma2c_nc_catchup.ini')['ENV_CONFIG']
    arrays, lines, _ = _run_oracle(cfg, str(tmp_path) + '/ref_')
    with caplog.at_level(logging.INFO):
        U.write_episode_records(U.split_episodes(0, *arrays), None, 'catchup', 'ma2c_nc', 0.1)
    assert [r.getMessage() for r in caplog.records if r.getMessage().startswith('test ')] == lines
    assert sorted(p.name for p in tmp_path.iterdir()) == ['ref_catchup_ma2c_nc_control.csv',
                                                          'ref_catchup_ma2c_nc_traffic.csv']
