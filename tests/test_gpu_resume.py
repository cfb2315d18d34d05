"""GPU: resuming batched training from a snapshot.

* One process, bit for bit: 3 updates, snapshot, 3 more updates (the reference) against fresh env / model / VecTrainer
  objects that restore the snapshot and run 3 updates, for every agent on both kernel families, with and without CUDA
  graphs.  Episodes of 2 updates, so per-env resets fall before and after the snapshot.  A catch-all compares every
  tensor attribute of the engine and the env right after the restore with the saved run's, except the scratch
  tensors the next update writes before it reads them.
* `main.py train` end to end: 6 updates in one run against 3 updates and a --resume raised to 6 updates (records
  byte for byte, final parameters and RMSProp state bit for bit, the same `evaluate` files); a configuration that
  differs in another key is refused.
* Changing the process count: a snapshot of two gloo ranks sharing the GPU restores into one process and the other
  way round, across the tensor-core / FFMA boundary (384 envs: 1 x 384 on tensor cores, 2 x 192 on FFMA).  Right after
  the restore the per-env state is the other side's, exactly; one update later the parameters and the record match
  the unchanged-count continuation up to summation order.  Two ranks resuming a two-rank snapshot end bit-identical.

Every child runs with a timeout; on timeout torchrun and every worker it started are stopped and the test fails.
"""
import configparser
import filecmp
import glob
import os
import sys

import numpy as np
import pytest
import torch

import resume_worker as W
from helpers import ROOT, load_cfg

pytestmark = pytest.mark.gpu
TIMEOUT = 900
PAR_KEYS = {'headway_target_range': '15, 25', 'speed_target_range': '12, 18', 'slowdown_prob': '0.5'}
SHORT = dict(episode_length_sec=12)          # 120 steps: an episode is 2 updates of 60


# ---- one process, bit for bit --------------------------------------------------------------------------------------
CASES = [('ma2c_nc', 'config_ma2c_nc_catchup.ini', 256, True, PAR_KEYS),
         ('ma2c_nc', 'config_ma2c_nc_catchup.ini', 200, False, {}),
         ('ma2c_dial', 'config_ma2c_dial_catchup.ini', 256, True, {}),
         ('ia2c', 'config_ia2c_catchup.ini', 130, False, PAR_KEYS),
         ('ia2c_fp', 'config_ia2c_fp_slowdown.ini', 128, None, {}),
         ('ma2c_cu', 'config_ia2c_cu_catchup.ini', 128, None, {})]


def _build(ini, n_env, over):
    import main
    from deeprl_network_b200 import utils as U
    cp = load_cfg(ini, n_env=n_env, **SHORT, **over)
    env = main.init_env(cp['ENV_CONFIG'])
    model = main.init_agent(env, cp['MODEL_CONFIG'], 10 ** 6, cp.getint('ENV_CONFIG', 'seed'))
    return env, model


def _tensors(obj):
    """{name: tensor} of every tensor attribute of obj, list elements as name[i]."""
    out = {}
    for k, v in vars(obj).items():
        if isinstance(v, torch.Tensor):
            out[k] = v
        elif isinstance(v, (list, tuple)):
            out.update({'%s[%d]' % (k, i): t for i, t in enumerate(v) if isinstance(t, torch.Tensor)})
    return out


# Written by the next update before it reads them: the ping-pong state slot 1, rollout slots 1..T, the rollout's
# actions / values / rewards / bootstrap, the returns, the learning-rate slot, gradients and optimizer scratch, the
# one-env API's staging, and the training buffers (allocated by the first update).
ENGINE_SCRATCH = {'c[1]', 'h[1]', 'msg[1]', 'act_buf', 'val_buf', 'rew_buf', 'grew_buf', 'R_end', 'boot_pi',
                  'boot_act', 'Rs', 'Advs', 'pi_tmp', 'lr_dev', 'grads', 'norm_out', 'opt_scratch', 'h_seq', 'c_seq',
                  'msg_seq', 'sv_xin', 'sv_sh', 'sv_gates', 'sv_enc', 'sv_dlv', 'sv_dz', 'sv_dpre', 'sv_dzT',
                  'sv_dpT', 'sv_dmp', 'dh_rec', 'dc_rec', 'dmsg', 'ws', 'loss_part', '_cu_scratch'}
SLOT0 = {'obs_buf', 'fp_buf', 'done_buf'}          # slot 0 is carried into the next update, slots 1..T are scratch
ENV_SCRATCH = {'_action_dev', '_u01'}


def _catch_all(saved, fresh, engine):
    scratch = set(ENGINE_SCRATCH)
    if not engine.use_tc or engine.variant == 'ma2c_dial':
        scratch.add('wt')          # the backward writes the transposed weights there (train.cu); elsewhere repack() does
    for name, a in saved['engine'].items():
        if name in scratch:
            continue
        b = fresh['engine'][name]
        if name in SLOT0:
            a, b = a[0], b[0]
        assert torch.equal(a, b), 'engine.' + name
    for name, a in saved['env'].items():
        if name not in ENV_SCRATCH:
            assert torch.equal(a, fresh['env'][name]), 'env.' + name


def _state(env, e, loop):
    em = (lambda t: t.permute(0, 2, 1)) if e.state_fm else (lambda t: t)
    out = dict(params=e.params, ms=e.ms, rng=e.rng, c=em(e.c[0]), h=em(e.h[0]), c_bw=em(e.c_bw), h_bw=em(e.h_bw),
               obs0=e.obs_buf[0], fp0=e.fp_buf[0], done0=e.done_buf[0], grew=e.grew_buf)
    if e.msg[0] is not None:
        out['msg'] = e.msg[0]
    out.update({'env.' + k: getattr(env, k) for k in env.SNAPSHOT_AXES if getattr(env, k) is not None})
    return {k: v.clone() for k, v in out.items()}


@pytest.mark.parametrize('graph', [True, False], ids=['graph', 'eager'])
@pytest.mark.parametrize('agent,ini,n_env,tc,over', CASES, ids=['%s_%d' % (c[0], c[2]) for c in CASES])
def test_restore_continues_bit_for_bit(agent, ini, n_env, tc, over, graph):
    from deeprl_network_b200 import utils as U
    env, model = _build(ini, n_env, over)
    loop = U.VecTrainer(env, model, graph=graph)
    loop.start()
    e = model.engine
    if tc is not None:
        assert e.use_tc == tc
    for _ in range(3):
        loop.update()
        loop.log_rewards(loop.n_update)
    snap = loop.snapshot()
    torch.cuda.synchronize()
    saved = dict(engine={k: v.clone() for k, v in _tensors(e).items()},
                 env={k: v.clone() for k, v in _tensors(env).items()})
    assert int(env.episode_dev.min()) >= 2                 # every env has been reset before the snapshot
    episodes = env.episode_dev.clone()
    for _ in range(3):
        loop.update()
        loop.log_rewards(loop.n_update)
    torch.cuda.synchronize()
    ref = _state(env, e, loop)
    assert bool((env.episode_dev > episodes).all())        # ... and after it
    ref_data = list(loop.data)
    loop.graph = None

    env2, model2 = _build(ini, n_env, over)
    loop2 = U.VecTrainer(env2, model2, graph=graph)
    loop2.start()
    loop2.restore(snap)
    torch.cuda.synchronize()
    _catch_all(saved, dict(engine=_tensors(model2.engine), env=_tensors(env2)), model2.engine)
    for _ in range(3):
        loop2.update()
        loop2.log_rewards(loop2.n_update)
    torch.cuda.synchronize()
    got = _state(env2, model2.engine, loop2)
    for k in ref:
        assert torch.equal(ref[k], got[k]), k
    assert loop2.data == ref_data and loop2.n_update == 6
    assert model2.lr_scheduler.n == model.lr_scheduler.n
    model2.engine.check_tc()
    loop2.graph = None


def test_linear_schedule_takes_the_new_horizon():
    """lr_decay = linear: after a resume with a larger total_step the rate is lr_init (1 - n / new total_step), n the
    env steps done -- a run that had reached lr_min at its old end goes back up and ramps down to the new end."""
    import main
    from deeprl_network_b200 import utils as U
    loops = []
    for total in (3, 6):                                        # updates of 60 steps x 128 envs
        cp = load_cfg('config_ma2c_nc_catchup.ini', n_env=128, **SHORT)
        cp['MODEL_CONFIG']['lr_decay'] = 'linear'
        lr_init, lr_min = cp.getfloat('MODEL_CONFIG', 'lr_init'), 0.1 * cp.getfloat('MODEL_CONFIG', 'lr_init')
        cp['MODEL_CONFIG']['lr_min'] = repr(lr_min)
        env = main.init_env(cp['ENV_CONFIG'])
        model = main.init_agent(env, cp['MODEL_CONFIG'], total * 60 * 128, cp.getint('ENV_CONFIG', 'seed'))
        loop = U.VecTrainer(env, model, graph=False)
        loop.start()
        loops.append(loop)
    first, longer = loops
    for _ in range(3):
        first.update()
    assert float(first.engine.lr_dev) == np.float32(lr_min)      # the first run ended at lr_min
    longer.restore(first.snapshot())
    longer.update()
    n = 4 * 60 * 128
    assert float(longer.engine.lr_dev) == np.float32(max(lr_min, lr_init * (1 - n / (6 * 60 * 128))))


# ---- main.py end to end ----------------------------------------------------------------------------------------------
def _run(cmd, env=None, ok=True):
    from deeprl_network_b200.dist import run_bounded
    rc, out = run_bounded(cmd, TIMEOUT, cwd=ROOT, env=env)
    if rc is None:
        pytest.fail('timed out after %d s, every process it started was stopped: %s\n%s'
                    % (TIMEOUT, ' '.join(cmd), out[-6000:]))
    if ok:
        assert rc == 0, '%s\nexit %d\n%s' % (' '.join(cmd), rc, out[-6000:])
    return rc, out


def _one_gpu_env():
    env = dict(os.environ)
    env['CUDA_VISIBLE_DEVICES'] = env.get('CUDA_VISIBLE_DEVICES', '0').split(',')[0] or '0'
    return env


def _ini(tmp, name, n_env, updates, interval_updates, file='exp.ini', model_over=None, **env_over):
    cp = configparser.ConfigParser()
    cp.read(os.path.join(ROOT, 'config', name))
    per = cp.getint('MODEL_CONFIG', 'batch_size') * n_env
    cp['TRAIN_CONFIG']['total_step'] = str(updates * per)
    cp['TRAIN_CONFIG']['log_interval'] = '1'
    cp['TRAIN_CONFIG']['greedy_test'] = 'true'
    cp['TRAIN_CONFIG']['checkpoint_interval'] = str(interval_updates * per)
    cp['ENV_CONFIG']['test_seeds'] = '10000,10010,10020'
    cp['ENV_CONFIG']['n_env'] = str(n_env)
    for k, v in dict(SHORT, **env_over).items():
        cp['ENV_CONFIG'][k] = str(v)
    for k, v in (model_over or {}).items():
        cp['MODEL_CONFIG'][k] = str(v)
    path = os.path.join(str(tmp), file)
    with open(path, 'w') as f:
        cp.write(f)
    return path


def _main(base, *args, procs=1, ok=True):
    main = os.path.join(ROOT, 'main.py')
    cmd = [sys.executable, main] if procs == 1 else \
        [sys.executable, '-m', 'torch.distributed.run', '--standalone', '--nproc-per-node', str(procs), main]
    return _run(cmd + ['--base-dir', base] + list(args), env=_one_gpu_env(), ok=ok)


def _files(base, pattern):
    return sorted(os.path.basename(f) for f in glob.glob(os.path.join(base, pattern)))


def test_cli_resume_matches_the_uninterrupted_run(tmp_path):
    ini, n_env = 'config_ma2c_nc_catchup.ini', 256
    per = 60 * n_env
    six = _ini(tmp_path, ini, n_env, 6, 3, **PAR_KEYS)
    a, b = str(tmp_path / 'a'), str(tmp_path / 'b')
    _main(a, 'train', '--config-dir', six)
    _main(b, 'train', '--config-dir', _ini(tmp_path, ini, n_env, 3, 3, file='short.ini', **PAR_KEYS))
    assert _files(b, 'model/*') == ['checkpoint-%d.pt' % (3 * per), 'resume-%d.pt' % (3 * per)]
    _, out = _main(b, 'train', '--config-dir', _ini(tmp_path, ini, n_env, 3, 3, file='other.ini',
                                                    model_over=dict(lr_init=1e-3), **PAR_KEYS), '--resume', ok=False)
    assert 'MODEL_CONFIG.lr_init' in out and 'ValueError' in out
    _main(b, 'train', '--config-dir', six, '--resume')
    assert _files(a, 'model/*') == _files(b, 'model/*') == [
        'checkpoint-%d.pt' % (3 * per), 'checkpoint-%d.pt' % (6 * per), 'resume-%d.pt' % (3 * per),
        'resume-%d.pt' % (6 * per)]
    assert _files(b, 'data/*.ini') == ['exp.ini']
    for f in ('train_reward.csv', 'env_par.csv', 'test_reward.csv'):
        assert filecmp.cmp(os.path.join(a, 'data', f), os.path.join(b, 'data', f), shallow=False), f
    ca, cb = (torch.load(os.path.join(d, 'model', 'checkpoint-%d.pt' % (6 * per))) for d in (a, b))
    assert torch.equal(ca['params'], cb['params']) and torch.equal(ca['ms'], cb['ms'])
    for d in (a, b):
        _main(d, 'evaluate', '--evaluation-seeds', '2000,2010')
    assert _files(a, 'eva_data/*') == _files(b, 'eva_data/*') and _files(a, 'eva_data/*')
    for f in _files(a, 'eva_data/*'):
        assert filecmp.cmp(os.path.join(a, 'eva_data', f), os.path.join(b, 'eva_data', f), shallow=False), f


def test_cli_two_ranks_resume_a_two_rank_snapshot(tmp_path):
    ini, n_env = 'config_ma2c_nc_catchup.ini', 256
    base = str(tmp_path / 'two')
    _main(base, 'train', '--config-dir', _ini(tmp_path, ini, n_env, 2, 2, **PAR_KEYS), procs=2)
    _main(base, 'train', '--config-dir', _ini(tmp_path, ini, n_env, 4, 2, **PAR_KEYS), '--resume', procs=2)
    logs = sorted(glob.glob(os.path.join(base, 'log', '*.log')), key=os.path.getmtime)
    assert 'bit-identical on all 2 ranks' in open(logs[-1]).read()
    assert len(open(os.path.join(base, 'data', 'train_reward.csv')).read().strip().split('\n')) == 5
    assert _files(base, 'model/resume-*') == ['resume-%d.pt' % (k * 60 * n_env) for k in (2, 4)]


# ---- changing the process count ----------------------------------------------------------------------------------------
def _worker(tmp, ini, before, after, snapshot=None):
    out = str(tmp)
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--standalone', '--nproc-per-node', '2',
           os.path.join(ROOT, 'tests', 'resume_worker.py'), ini, out, str(before), str(after)]
    _run(cmd + ([snapshot] if snapshot else []), env=_one_gpu_env())
    return out


def _close(a, b):
    """Equal up to the order of the gradient sums and the kernel path: each tensor against its own scale, as
    test_gpu_dist_train.py judges it, with 1e-4 instead of 1e-5 because the two sides also run different kernels
    (3xTF32 tensor cores on one, FP32 FFMA on the other), which round differently."""
    a, b = a.double(), b.double()
    assert float((a - b).abs().max()) <= 1e-4 * max(float(a.abs().max()), 1e-6)


def _close_params(end, e):
    from deeprl_network_b200.envs.cacc_env import chain_masks
    from deeprl_network_b200.layout import ModelLayout
    for name, o, shape in ModelLayout('ma2c_nc', [5] * 8, 4, chain_masks(8)[0]).entries:
        n = int(np.prod(shape))
        for key in ('params', 'ms'):
            _close(end[key][o:o + n], getattr(e, key).cpu()[o:o + n])


def _close_record(a, b):
    assert a['step'] == b['step']
    # the rollout's policies differ in the last bits between the kernel paths (test_reward's tolerance there)
    np.testing.assert_allclose([b['avg_reward'], b['std_reward']], [a['avg_reward'], a['std_reward']], rtol=1e-3)


N_ENV = 384                  # one process: 384 envs on tensor cores; two ranks: 192 each on FFMA


def _pc_ini(tmp):
    return _ini(tmp, 'config_ma2c_nc_catchup.ini', N_ENV, 10, 10, **PAR_KEYS)


def test_two_rank_snapshot_restores_into_one_process(tmp_path):
    ini = _pc_ini(tmp_path)
    out = _worker(tmp_path, ini, 3, 1)
    snap = torch.load(os.path.join(out, 'snap.pt'), weights_only=True)
    parts = [torch.load(os.path.join(out, 'local-%d.pt' % r), weights_only=True) for r in range(2)]
    whole = W.snapshot_state(snap)
    loop = W.build(ini)
    assert loop.engine.use_tc
    _, axes = W.local_state(loop)
    for k, v in whole.items():
        assert torch.equal(v, torch.cat([p[k] for p in parts], dim=axes[k])), k
    loop.restore(snap)
    mine, _ = W.local_state(loop)
    assert mine.keys() == whole.keys()
    for k in whole:
        assert torch.equal(mine[k], whole[k]), k
    W.run(loop, 1)
    end = torch.load(os.path.join(out, 'end.pt'), weights_only=True)
    _close_params(end, loop.engine)
    assert len(loop.data) == len(end['data']) == 4
    _close_record(end['data'][-1], loop.data[-1])
    loop.graph = None


def test_one_process_snapshot_restores_into_two_ranks(tmp_path):
    from deeprl_network_b200 import dist as D
    ini = _pc_ini(tmp_path)
    loop = W.build(ini)
    W.run(loop, 3)
    snap = loop.snapshot()
    path = os.path.join(str(tmp_path), 'snap.pt')
    torch.save(snap, path)
    W.run(loop, 1)
    loop.graph = None
    out = _worker(tmp_path, ini, 0, 1, path)
    whole = W.snapshot_state(snap)
    _, axes = W.local_state(loop)
    for r in range(2):
        got = torch.load(os.path.join(out, 'restored-%d.pt' % r), weights_only=True)
        want = D.take_envs(whole, axes, *D.env_shard(N_ENV, 2, r))
        assert got.keys() == want.keys()
        for k in want:
            assert torch.equal(got[k], want[k]), (r, k)
    end = torch.load(os.path.join(out, 'end.pt'), weights_only=True)
    _close_params(end, loop.engine)
    assert len(end['data']) == len(loop.data) == 4
    _close_record(loop.data[-1], end['data'][-1])
