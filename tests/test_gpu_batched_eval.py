"""GPU: greedy evaluation episodes batched on the device (BatchedEvaluator, nmarl_eval_record).

* `main.py evaluate`'s batched path writes the same bytes as the one-seed-at-a-time Evaluator: all six agents,
  catch-up and slow-down, 12 seeds and 130 seeds (not a multiple of 128, in one pass and in passes of 64).
* `main.py train` + `evaluate` with the default 50 seeds writes what the Evaluator writes for that checkpoint.
* TRAIN_CONFIG.greedy_test: one test_reward.csv row per log record, equal to B = 1 greedy episodes on the same
  weights; with the key off nothing changes, and with it on the training state is the same as with it off.
* The recorder, fed the reference's actions, reproduces the reference env's CSV files (tests/golden/eval_*).
"""
import configparser
import os

import numpy as np
import pytest
import torch

import main
from deeprl_network_b200 import _lib as L
from deeprl_network_b200 import utils as U
from deeprl_network_b200.envs.cacc_env import CACCEnv
from helpers import GOLDEN, ROOT, load_cfg, random_params

pytestmark = pytest.mark.gpu

CONFIGS = {('ia2c', 'catchup'): 'config_ia2c_catchup.ini', ('ia2c', 'slowdown'): 'config_ia2c_slowdown.ini',
           ('ia2c_fp', 'catchup'): 'config_ia2c_fp_catchup.ini', ('ia2c_fp', 'slowdown'): 'config_ia2c_fp_slowdown.ini',
           ('ma2c_cu', 'catchup'): 'config_ia2c_cu_catchup.ini', ('ma2c_cu', 'slowdown'): 'config_ia2c_cu_slowdown.ini',
           ('ma2c_nc', 'catchup'): 'config_ma2c_nc_catchup.ini', ('ma2c_nc', 'slowdown'): 'config_ma2c_nc_slowdown.ini',
           ('ma2c_ic3', 'catchup'): 'config_ma2c_cnet_catchup.ini',
           ('ma2c_ic3', 'slowdown'): 'config_ma2c_cnet_slowdown.ini',
           ('ma2c_dial', 'catchup'): 'config_ma2c_dial_catchup.ini',
           ('ma2c_dial', 'slowdown'): 'config_ma2c_dial_slowdown.ini'}
SEEDS12 = list(range(2000, 2120, 10))


def _one_env_model(cp, seed=3):
    """n_env = 1 env + agent (what main.evaluate builds) with random weights.  The policy bias leans towards
    action 0 (no acceleration command), so that slow-down platoons collide and some episodes end early."""
    cp['ENV_CONFIG']['n_env'] = '1'
    env = CACCEnv(cp['ENV_CONFIG'])
    model = main.init_agent(env, cp['MODEL_CONFIG'], 0, 0)
    w = random_params(model.layout.creation_order(), seed=seed, scale=1.0)
    for name, _, shape in model.layout.entries:
        if '/pi' in name and name.endswith('/b'):
            w[name] = w[name] + np.array([1.5, 0, 0, 0], dtype=np.float32)
    model.set_weights(w)
    return env, model


def _per_seed(env, model, seeds, out):
    env.init_test_seeds(seeds)
    U.Evaluator(env, model, out).run()


def _read(d):
    return {f: open(os.path.join(d, f), 'rb').read() for f in sorted(os.listdir(d))}


def _episode_lengths(d):
    import pandas as pd
    ctl = pd.read_csv([os.path.join(d, f) for f in os.listdir(d) if f.endswith('_control.csv')][0])
    return ctl.groupby('episode').size().values


@pytest.mark.parametrize('scenario', ['catchup', 'slowdown'])
@pytest.mark.parametrize('agent', ['ia2c', 'ia2c_fp', 'ma2c_cu', 'ma2c_nc', 'ma2c_ic3', 'ma2c_dial'])
def test_batched_evaluate_is_byte_identical(agent, scenario, tmp_path):
    cp = load_cfg(CONFIGS[agent, scenario])
    env, model = _one_env_model(cp)
    one, many = str(tmp_path / 'one') + '/', str(tmp_path / 'many') + '/'
    os.makedirs(one), os.makedirs(many)
    _per_seed(env, model, SEEDS12, one)
    params = model.engine.params.clone()
    ev = U.BatchedEvaluator(cp['ENV_CONFIG'], model, many)
    ev.run(SEEDS12)
    assert _read(many) == _read(one)
    assert len(_read(one)) == 2
    assert torch.equal(model.engine.params, params) and ev._runners[12]['eng'].params is model.engine.params
    assert not ev._runners[12]['eng'].use_tc
    lengths = _episode_lengths(one)
    assert len(lengths) == 12
    if scenario == 'slowdown':
        assert (lengths < env.T).any(), 'no episode ended before T'


def test_batched_evaluate_130_seeds_in_passes(tmp_path):
    """130 envs in one pass, and in passes of 64, 64 and 2 (the second 64-env pass replays a CUDA graph)."""
    cp = load_cfg(CONFIGS['ma2c_nc', 'slowdown'])
    env, model = _one_env_model(cp, seed=5)
    seeds = list(range(3000, 3000 + 130))
    one = str(tmp_path / 'one') + '/'
    os.makedirs(one)
    _per_seed(env, model, seeds, one)
    ref = _read(one)
    lengths = _episode_lengths(one)
    assert (lengths < env.T).any() and len(lengths) == 130
    for max_env, graph in ((4096, True), (64, True), (64, False)):
        out = str(tmp_path / ('many%d%d' % (max_env, graph))) + '/'
        os.makedirs(out)
        ev = U.BatchedEvaluator(cp['ENV_CONFIG'], model, out, max_env=max_env, graph=graph)
        ev.run(seeds)
        assert _read(out) == ref, (max_env, graph)
        if max_env == 64:
            assert sorted(ev._runners) == [2, 64]
            assert (ev._runners[64]['graph'] is not None) == graph


def _write_cfg(tmp_path, ini, env_over=(), train_over=()):
    cp = configparser.ConfigParser()
    assert cp.read(os.path.join(ROOT, 'config', ini))
    for k, v in dict(env_over).items():
        cp['ENV_CONFIG'][k] = str(v)
    for k, v in dict(train_over).items():
        cp['TRAIN_CONFIG'][k] = str(v)
    path = str(tmp_path / ('%s.ini' % os.path.basename(str(tmp_path))))
    with open(path, 'w') as f:
        cp.write(f)
    return path


def test_cli_evaluate_matches_per_seed_evaluator(tmp_path):
    """main.py train (batched) then main.py evaluate with the default 50 seeds == the Evaluator on that checkpoint."""
    n_env = 16
    ini = _write_cfg(tmp_path, 'config_ia2c_fp_catchup.ini', dict(n_env=n_env),
                     dict(total_step=2 * 60 * n_env, log_interval=60 * n_env))
    base = str(tmp_path / 'run')
    main.train(main.parse_args(['--base-dir', base, 'train', '--config-dir', ini]))
    main.evaluate(main.parse_args(['--base-dir', base, 'evaluate']))
    seeds = [int(s) for s in main.DEFAULT_EVAL_SEEDS.split(',')]
    assert len(seeds) == 50
    # the parent commit's evaluate: one env, one seed after the other
    cfg = main.read_config(U.find_file(base + '/data/'))
    cfg['ENV_CONFIG']['n_env'] = '1'
    env = main.init_env(cfg['ENV_CONFIG'])
    model = main.init_agent(env, cfg['MODEL_CONFIG'], 0, 0)
    assert model.load(base + '/model/')
    ref = str(tmp_path / 'ref') + '/'
    os.makedirs(ref)
    _per_seed(env, model, seeds, ref)
    got = {f: b for f, b in _read(base + '/eva_data').items() if f.endswith('.csv')}
    assert got == _read(ref) and len(got) == 2


class _SnapshotEvaluator(U.BatchedEvaluator):
    """BatchedEvaluator that keeps the weights it evaluated at each record."""
    made = []

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.snaps = []
        _SnapshotEvaluator.made.append(self)

    def log_test(self, global_step, seeds, summary_writer=None):
        self.snaps.append(self.model.engine.params.clone())
        return super().log_test(global_step, seeds, summary_writer)


def _host_greedy_rewards(ini, params, seeds):
    """Trainer.perform's B = 1 greedy episodes, one seed after the other, on these weights: the per-step global
    rewards of all episodes in seed order."""
    cfg = main.read_config(ini)
    cfg['ENV_CONFIG']['n_env'] = '1'
    env = main.init_env(cfg['ENV_CONFIG'])
    env.init_test_seeds(seeds)
    model = main.init_agent(env, cfg['MODEL_CONFIG'], 0, 0)
    model.engine.params.copy_(params)
    model.engine.repack(); model.engine._refresh_msg()
    rewards, step = [], env.step

    def recording_step(action):
        out = step(action)
        rewards.append(out[3])
        return out
    env.step = recording_step
    ev = U.Evaluator(env, model, None)
    for k in range(len(seeds)):
        ev.perform(k)
    return np.array(rewards)


@pytest.mark.parametrize('ini', ['config_ma2c_dial_slowdown.ini', 'config_ia2c_catchup.ini'])
def test_greedy_test_records(tmp_path, monkeypatch, ini):
    import pandas as pd
    n_env, seeds = 128, SEEDS12[:5]
    path = _write_cfg(tmp_path, ini, dict(n_env=n_env, test_seeds=','.join(map(str, seeds))),
                      dict(total_step=3 * 60 * n_env, log_interval=60 * n_env, greedy_test='true'))
    _SnapshotEvaluator.made = []
    monkeypatch.setattr(U, 'BatchedEvaluator', _SnapshotEvaluator)
    base = str(tmp_path / 'run')
    main.train(main.parse_args(['--base-dir', base, 'train', '--config-dir', path]))
    train = pd.read_csv(base + '/data/train_reward.csv')
    test = pd.read_csv(base + '/data/test_reward.csv', float_precision='round_trip')
    assert list(test.columns)[1:] == ['agent', 'step', 'test_id', 'avg_reward', 'std_reward']
    assert len(test) == len(train) == 3 and list(test['step']) == list(train['step'])
    (ev,) = _SnapshotEvaluator.made
    assert len(ev.snaps) == 3 and not torch.equal(ev.snaps[0], ev.snaps[2])
    for k, snap in enumerate(ev.snaps):
        r = _host_greedy_rewards(path, snap, seeds)
        assert ev.data[k]['avg_reward'] == np.mean(r) and ev.data[k]['std_reward'] == np.std(r), k
        assert test['avg_reward'][k] == np.mean(r) and test['std_reward'][k] == np.std(r), k


def test_greedy_test_off_changes_nothing(tmp_path):
    n_env = 128
    runs = {}
    for key in (None, 'false'):
        over = dict(total_step=2 * 60 * n_env, log_interval=60 * n_env)
        if key is not None:
            over['greedy_test'] = key
        d = tmp_path / str(key)
        d.mkdir()
        path = _write_cfg(d, 'config_ma2c_nc_catchup.ini', dict(n_env=n_env), over)
        base = str(d / 'run')
        main.train(main.parse_args(['--base-dir', base, 'train', '--config-dir', path]))
        runs[key] = sorted(os.listdir(base + '/data'))
        runs[key, 'csv'] = open(base + '/data/train_reward.csv', 'rb').read()
    assert 'test_reward.csv' not in runs['false'] and 'test_reward.csv' not in runs[None]
    assert runs[None, 'csv'] == runs['false', 'csv']


def _training_state(graph, greedy, n_update=3):
    cp = load_cfg('config_ma2c_nc_catchup.ini', n_env=128, test_seeds=','.join(map(str, SEEDS12[:4])))
    env = main.init_env(cp['ENV_CONFIG'])
    model = main.init_agent(env, cp['MODEL_CONFIG'], 10 ** 6, 12)
    loop = U.VecTrainer(env, model, graph=graph)
    loop.start()
    tester = U.BatchedEvaluator(cp['ENV_CONFIG'], model) if greedy else None
    rewards = []
    for k in range(n_update):
        loop.update()
        rewards.append(loop.log_rewards(k))
        if tester is not None:
            tester.log_test(k, env.test_seeds)
    torch.cuda.synchronize()
    e = model.engine
    state = dict(params=e.params, ms=e.ms, rng=e.rng, grew=e.grew_buf, c=e.c[e.cur], h=e.h[e.cur], c_bw=e.c_bw,
                 h_bw=e.h_bw, obs=e.obs_buf, fp=e.fp_buf, done=e.done_buf, hs=env.hs, vs=env.vs, us=env.us,
                 t=env.t_dev, episode=env.episode_dev)
    return {k: v.clone() for k, v in state.items()}, rewards, np.random.get_state()[1].copy()


@pytest.mark.parametrize('graph', [False, True], ids=['eager', 'graph'])
def test_greedy_test_does_not_perturb_training(graph):
    off, r_off, rng_off = _training_state(graph, False)
    on, r_on, rng_on = _training_state(graph, True)
    assert r_on == r_off
    for k in off:
        assert torch.equal(on[k], off[k]), k
    np.testing.assert_array_equal(rng_on, rng_off)


def test_recorder_reproduces_reference_csv(tmp_path):
    """The reference env's files for the recorded actions (same bar as test_evaluator_csv_matches_reference): 33
    envs (two recorder blocks) all take the reference's actions; env 0 and env 32 are written out."""
    import pandas as pd
    cp = load_cfg('config_ma2c_nc_catchup.ini')
    E = 33
    env = CACCEnv(cp['ENV_CONFIG'], n_env=E)
    env.train_mode = False
    acts = np.load(GOLDEN + '/eval_actions.npy')
    T, N = env.T, env.n_agent
    dev = env.device
    np.random.seed(2000)
    env.reset_device(u01=torch.full((1, E), np.random.rand(), dtype=torch.float64, device=dev))
    z = lambda *s, dtype=torch.float64: torch.zeros(*s, dtype=dtype, device=dev)
    alive, steps = z(E, dtype=torch.int32), z(E, dtype=torch.int32)
    rec = dict(action=z(T + 1, E, N, dtype=torch.int32), reward=z(T + 1, E), hs=z(T + 1, E, N), vs=z(T + 1, E, N),
               us=z(T + 1, E, N))
    act = z(N, E, dtype=torch.int32)

    def record(start):
        L.check(L.lib().nmarl_eval_record(N, E, T, start, L.ptr(act), L.ptr(env.greward_dev), L.ptr(env.done_dev),
                                          L.ptr(env.hs), L.ptr(env.vs), L.ptr(env.us), L.ptr(alive), L.ptr(steps),
                                          L.ptr(rec['action']), L.ptr(rec['reward']), L.ptr(rec['hs']),
                                          L.ptr(rec['vs']), L.ptr(rec['us']), L.stream()), 'nmarl_eval_record')
    record(1)
    for t in range(len(acts)):
        act.copy_(torch.as_tensor(np.asarray(acts[t], dtype=np.int32))[:, None].expand(-1, E))
        env.step_device(act)
        record(0)
    host = [steps.cpu().numpy()] + [rec[k].cpu().numpy() for k in ('action', 'reward', 'hs', 'vs', 'us')]
    assert (host[0] == len(acts)).all() and not alive.any()
    for b in (0, 32):
        out = str(tmp_path / str(b)) + '/'
        os.makedirs(out)
        one = [host[0][b:b + 1]] + [a[:, b:b + 1] for a in host[1:]]
        U.write_episode_records(U.split_episodes(0, *one), out, 'catchup', 'ma2c_nc', env.dt)
        for kind in ('control', 'traffic'):
            mine = pd.read_csv(out + 'catchup_ma2c_nc_%s.csv' % kind)
            ref = pd.read_csv(GOLDEN + '/eval_catchup_ma2c_nc_%s.csv' % kind)
            assert list(mine.columns) == list(ref.columns)
            assert len(mine) == len(ref)
            for col in ref.columns:
                if not pd.api.types.is_numeric_dtype(ref[col]):
                    assert (mine[col] == ref[col]).all(), col
                else:
                    np.testing.assert_allclose(mine[col].values, ref[col].values, rtol=1e-9, atol=1e-9, err_msg=col)
