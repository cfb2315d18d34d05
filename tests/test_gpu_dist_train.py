"""GPU: training one configuration on several processes.

* Keying: a shard holding the global envs env0 .. env0 + B - 1 of B_total resets, draws its per-env parameters, steps
  and samples exactly what those envs of one process holding all B_total do, on the tensor-core and the FFMA kernels.
* `main.py train` under torchrun, two ranks sharing one GPU (gloo), against the one-process run of the same .ini over
  one update: train_reward.csv and env_par.csv byte for byte, the checkpoint up to summation order, test_reward.csv
  within 1e-3 relative.  Over three updates both ranks end with bit-identical parameters and RMSProp state (main.py
  checks it and exits non-zero otherwise).  The same parity with NCCL and CUDA graphs needs two GPUs.

Every child runs with a timeout; on timeout torchrun and every worker it started are stopped and the test fails.
"""
import configparser
import glob
import os
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT, load_cfg

pytestmark = pytest.mark.gpu
TIMEOUT = 900
PAR_KEYS = {'headway_target_range': '15, 25', 'speed_target_range': '12, 18', 'slowdown_prob': '0.5'}


# ---- keying ---------------------------------------------------------------------------------------------------------
def _pair(agent, scen, total, local, env0, **env_over):
    from deeprl_network_b200.agents.models import IA2C, MA2C_DIAL, MA2C_NC
    from deeprl_network_b200.envs.cacc_env import CACCEnv
    cls = {'ma2c_nc': MA2C_NC, 'ma2c_dial': MA2C_DIAL, 'ia2c': IA2C}[agent]
    out = []
    for B, e0 in ((total, 0), (local, env0)):
        cp = load_cfg('config_%s_%s.ini' % (agent, scen), n_env=total, **env_over)
        env = CACCEnv(cp['ENV_CONFIG'], n_env=B, env0=e0, n_env_total=total)
        kw = dict(obs_mode='gather') if agent == 'ia2c' else {}
        model = cls(env.n_s_ls, env.n_a_ls, env.neighbor_mask, env.distance_mask, env.coop_gamma, 10 ** 6,
                    cp['MODEL_CONFIG'], seed=12, n_env=B, env0=e0, n_env_total=total, **kw)
        out.append((env, model))
    return out


@pytest.mark.parametrize('agent,scen,total,local,env0,tc', [
    ('ma2c_nc', 'catchup', 256, 128, 128, True),
    ('ma2c_dial', 'catchup', 256, 128, 128, True),
    ('ma2c_nc', 'catchup', 130, 65, 65, False),
    ('ia2c', 'slowdown', 130, 65, 65, False)])
def test_shard_rollout_is_the_one_process_rollout(agent, scen, total, local, env0, tc):
    """First rollout (reset, p-calls with Philox sampling, v-calls, env steps, bootstrap) of the shard == rows
    env0 .. env0 + local - 1 of the one-process rollout, bit for bit."""
    (env_a, mod_a), (env_b, mod_b) = _pair(agent, scen, total, local, env0, **PAR_KEYS)
    ea, eb = mod_a.engine, mod_b.engine
    assert ea.use_tc == eb.use_tc == tc
    assert torch.equal(ea.params, eb.params)
    for env, e in ((env_a, ea), (env_b, eb)):
        env.reset_device(u01=None, philox_seed=env.seed)
        e.reset_states()
        e.begin_episode(env)
        e.rollout(env)
    torch.cuda.synchronize()
    sl = slice(env0, env0 + local)
    for name in ('act_buf', 'obs_buf', 'fp_buf', 'val_buf', 'grew_buf', 'rew_buf', 'done_buf', 'boot_act', 'R_end'):
        a, b = getattr(ea, name), getattr(eb, name)
        dim = a.dim() - 2 if name in ('obs_buf', 'fp_buf') else a.dim() - 1
        assert torch.equal(a.narrow(dim, env0, local), b), name
    assert torch.equal(env_a.env_par[sl], env_b.env_par)
    ea.check_tc(); eb.check_tc()


def test_shard_env_is_the_one_process_env():
    """600 steps of random actions with per-env resets (new episode counters, new parameter rows): env0 = 64 of 128
    holds exactly envs 64..127 of the 128-env env."""
    from deeprl_network_b200.envs.cacc_env import CACCEnv
    cp = load_cfg('config_ma2c_nc_catchup.ini', n_env=128, batch_size=20, episode_length_sec=10, **PAR_KEYS)
    full = CACCEnv(cp['ENV_CONFIG'])
    part = CACCEnv(cp['ENV_CONFIG'], n_env=64, env0=64, n_env_total=128)
    sl = slice(64, 128)
    rng = np.random.default_rng(3)
    for env in (full, part):
        env.reset_device(philox_seed=env.seed)
    for step in range(600):
        act = torch.as_tensor(rng.integers(0, 4, size=(full.n_agent, 128), dtype=np.int32)).cuda()
        full.step_device(act)
        part.step_device(act[:, sl].contiguous())
        for env in (full, part):
            env.reset_device(mask=env.done_dev.clone(), philox_seed=env.seed)
        if step % 50 == 49 or step == 599:
            for name in ('hs', 'vs', 'us', 'v_init', 'reward_dev'):
                assert torch.equal(getattr(full, name)[:, sl], getattr(part, name)), (step, name)
            for name in ('t_dev', 'collision_dev', 'episode_dev', 'greward_dev', 'done_dev', 'env_par'):
                assert torch.equal(getattr(full, name)[sl], getattr(part, name)), (step, name)
            assert torch.equal(full.obs_dev[:, sl], part.obs_dev)
    assert int(part.episode_dev.min()) >= 6           # every env went through several resets


# ---- main.py train under torchrun ------------------------------------------------------------------------------------
def _run(cmd, env=None):
    """Run a child with a timeout (dist.run_bounded: on timeout torchrun and every worker it started are stopped, and
    the test fails); the child must exit with status 0."""
    from deeprl_network_b200.dist import run_bounded
    rc, out = run_bounded(cmd, TIMEOUT, cwd=ROOT, env=env)
    if rc is None:
        pytest.fail('timed out after %d s, every process it started was stopped: %s\n%s'
                    % (TIMEOUT, ' '.join(cmd), out[-6000:]))
    assert rc == 0, '%s\nexit %d\n%s' % (' '.join(cmd), rc, out[-6000:])
    return out


def _ini(tmp, name, updates, **env_over):
    cp = configparser.ConfigParser()
    cp.read(os.path.join(ROOT, 'config', name))
    n_env = int(env_over['n_env'])
    T = cp.getint('MODEL_CONFIG', 'batch_size')
    cp['TRAIN_CONFIG']['total_step'] = str(updates * T * n_env)
    cp['TRAIN_CONFIG']['log_interval'] = '1'
    cp['TRAIN_CONFIG']['greedy_test'] = 'true'
    cp['ENV_CONFIG']['test_seeds'] = '10000,10010,10020'
    for k, v in env_over.items():
        cp['ENV_CONFIG'][k] = str(v)
    path = os.path.join(str(tmp), 'exp.ini')
    with open(path, 'w') as f:
        cp.write(f)
    return path


def _train(tmp, tag, ini, procs=1, env=None):
    base = os.path.join(str(tmp), tag)
    main = os.path.join(ROOT, 'main.py')
    cmd = [sys.executable, main] if procs == 1 else \
        [sys.executable, '-m', 'torch.distributed.run', '--standalone', '--nproc-per-node', str(procs), main]
    _run(cmd + ['--base-dir', base, 'train', '--config-dir', ini], env=env)
    return base


def _one_gpu_env():
    env = dict(os.environ)
    first = env.get('CUDA_VISIBLE_DEVICES', '0').split(',')[0] or '0'
    env['CUDA_VISIBLE_DEVICES'] = first
    return env


def _checkpoint(base):
    files = glob.glob(os.path.join(base, 'model', 'checkpoint-*.pt'))
    assert len(files) == 1, files
    return torch.load(files[0], map_location='cpu')


def _compare(one, many, agent, par):
    for f in ['train_reward.csv'] + (['env_par.csv'] if par else []):
        assert open(os.path.join(one, 'data', f), 'rb').read() == open(os.path.join(many, 'data', f), 'rb').read(), f
    # the gradient is summed in another order: judge each tensor against its own scale
    ca, cb = _checkpoint(one), _checkpoint(many)
    assert ca['global_step'] == cb['global_step'] and ca['names'] == cb['names']
    entries = _entries(agent)
    for name, o, shape in entries:
        n = int(np.prod(shape))
        for key in ('params', 'ms'):
            a, b = ca[key][o:o + n].double(), cb[key][o:o + n].double()
            scale = float(a.abs().max())
            assert float((a - b).abs().max()) <= 1e-5 * max(scale, 1e-6), (key, name)
    ta = np.loadtxt(os.path.join(one, 'data', 'test_reward.csv'), delimiter=',', skiprows=1, usecols=(4, 5))
    tb = np.loadtxt(os.path.join(many, 'data', 'test_reward.csv'), delimiter=',', skiprows=1, usecols=(4, 5))
    np.testing.assert_allclose(tb, ta, rtol=1e-3)


def _entries(agent):
    """(name, offset, shape) of every tensor of the 8-vehicle platoon model's flat parameter buffer"""
    from deeprl_network_b200.envs.cacc_env import chain_masks
    from deeprl_network_b200.layout import ModelLayout
    nb, _ = chain_masks(8)
    n_s = [5] * 8 if agent.startswith('ma2c') else [5 * (1 + int(nb[i].sum())) for i in range(8)]
    return ModelLayout(agent, n_s, 4, nb, obs_mode='gather').entries


CASES = [('ma2c_nc', 'config_ma2c_nc_catchup.ini', dict(n_env=256, **PAR_KEYS)),       # tensor cores, 128 per rank
         ('ma2c_dial', 'config_ma2c_dial_catchup.ini', dict(n_env=256)),               # env-major state
         ('ia2c', 'config_ia2c_slowdown.ini', dict(n_env=130))]                        # FFMA, 65 per rank


@pytest.mark.parametrize('agent,ini,over', CASES, ids=[c[0] for c in CASES])
def test_cli_two_ranks_on_one_gpu_match_one_process(tmp_path, agent, ini, over):
    path = _ini(tmp_path, ini, 1, **over)
    env = _one_gpu_env()
    one = _train(tmp_path, 'one', path, 1, env)
    two = _train(tmp_path, 'two', path, 2, env)
    _compare(one, two, agent, 'slowdown_prob' in over)
    assert sorted(os.listdir(os.path.join(two, 'data'))) == sorted(os.listdir(os.path.join(one, 'data')))


def test_cli_two_ranks_keep_identical_replicas(tmp_path):
    path = _ini(tmp_path, 'config_ma2c_nc_catchup.ini', 3, n_env=256, **PAR_KEYS)
    base = _train(tmp_path, 'two', path, 2, _one_gpu_env())
    log = ''.join(open(f).read() for f in glob.glob(os.path.join(base, 'log', '*.log')))
    assert 'bit-identical on all 2 ranks' in log
    assert len(open(os.path.join(base, 'data', 'train_reward.csv')).read().strip().split('\n')) == 4


def test_cli_nccl_with_graphs_matches_one_process(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip('NCCL parity not run: it needs two GPUs, this machine has %d' % torch.cuda.device_count())
    agent, ini, over = CASES[0]
    path = _ini(tmp_path, ini, 1, **over)
    one = _train(tmp_path, 'one', path, 1, _one_gpu_env())
    two = _train(tmp_path, 'two', path, 2, dict(os.environ))
    log = ''.join(open(f).read() for f in glob.glob(os.path.join(two, 'log', '*.log')))
    assert '(nccl)' in log
    _compare(one, two, agent, True)
