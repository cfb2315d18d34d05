"""CPU: training on several processes without a GPU -- which envs and test seeds a rank owns, how many environment
steps an update counts, every refusal, the sampling-lane checks of the C ABI, and that the records rank 0 computes from
the gathered per-rank arrays are byte-identical to the one-process records."""
import ctypes
import types

import numpy as np
import pytest
import torch

import main
from deeprl_network_b200 import _lib as L
from deeprl_network_b200 import dist as D
from deeprl_network_b200 import utils as U
from deeprl_network_b200.envs.cacc_env import CACCEnv
from helpers import ROOT  # noqa: F401  (puts the repository on sys.path)

WORLDS = [1, 2, 3, 8]


@pytest.mark.parametrize('world', WORLDS)
def test_env_shards_tile_the_global_envs_in_order(world):
    n_env = 24 * world
    got = [D.env_shard(n_env, world, r) for r in range(world)]
    assert all(n == n_env // world for _, n in got)
    assert np.array_equal(np.concatenate([np.arange(e0, e0 + n) for e0, n in got]), np.arange(n_env))


@pytest.mark.parametrize('world', WORLDS)
@pytest.mark.parametrize('n_seed', [1, 3, 50])
def test_seed_shards_are_contiguous_and_cover_every_seed_once(world, n_seed):
    seeds = list(range(2000, 2000 + 10 * n_seed, 10))
    parts = [D.seed_shard(seeds, world, r) for r in range(world)]
    assert sum(parts, []) == seeds
    assert max(map(len, parts)) - min(map(len, parts)) <= 1


@pytest.mark.parametrize('world', [2, 3, 8])
def test_refusals(world):
    with pytest.raises(ValueError, match='multiple'):
        D.env_shard(8 * world + 1, world, 0)
    with pytest.raises(ValueError, match='one-env Trainer'):
        D.env_shard(1, world, world - 1)
    assert D.env_shard(1, 1, 0) == (0, 1)


def _ini(tmp_path, n_env):
    import configparser
    import os
    cp = configparser.ConfigParser()
    cp.read(os.path.join(ROOT, 'config', 'config_ma2c_nc_catchup.ini'))
    cp['ENV_CONFIG']['n_env'] = str(n_env)
    path = tmp_path / 'exp.ini'
    with open(path, 'w') as f:
        cp.write(f)
    return str(path)


@pytest.mark.parametrize('n_env', [1, 7])
def test_train_refuses_before_the_process_group_exists(tmp_path, monkeypatch, n_env):
    monkeypatch.setenv('WORLD_SIZE', '2')
    monkeypatch.setenv('RANK', '1')
    monkeypatch.setattr(D, 'init_from_env', lambda: pytest.fail('process group initialised before the refusal'))
    with pytest.raises(ValueError):
        main.train(main.parse_args(['--base-dir', str(tmp_path / 'run'), 'train', '--config-dir', _ini(tmp_path, n_env)]))
    assert not (tmp_path / 'run').exists()


def test_evaluate_refuses_several_processes(tmp_path, monkeypatch):
    monkeypatch.setenv('WORLD_SIZE', '2')
    with pytest.raises(ValueError, match='one process'):
        main.evaluate(main.parse_args(['--base-dir', str(tmp_path), 'evaluate', '--evaluation-seeds', '2000']))


class _Loop:
    def __init__(self, env, model, graph=True):
        self.n_update, self.graph = 0, graph

    def start(self):
        pass

    def update(self):
        self.n_update += 1

    def log_rewards(self, step, writer):
        return None


@pytest.mark.parametrize('world', WORLDS)
def test_an_update_counts_the_steps_of_every_env_of_every_rank(world, monkeypatch):
    monkeypatch.setattr(U, 'VecTrainer', _Loop)
    T, total = 60, 128 * world
    env = types.SimpleNamespace(n_env=total // world, n_env_total=total, test_seeds=[])
    model = types.SimpleNamespace(n_step=T)
    done = main._train_batched(env, model, 5 * T * total, 1)
    assert done == 5 * T * total


# ---- the sampling-lane and shard checks of the C ABI (before any launch: no GPU needed) --------------------------------
def _fwd(B, env0, B_total):
    a = L.FwdArgs()
    a.B, a.env0, a.B_total = B, env0, B_total
    for f in ('params', 'obs', 'fp', 'done', 'c_in', 'h_in', 'c_out', 'h_out', 'msg_in', 'msg_out'):
        setattr(a, f, 16 + 16 * len(f))                      # never dereferenced: the call is refused first
    a.sample_mode = L.SAMPLE_NONE
    return a


def test_policy_step_p_refuses_lanes_outside_the_run():
    from test_host_layout import _layout
    lay, _, _ = _layout('ma2c_nc')
    m, lib = lay.c_model(), L.lib()
    for env0, B_total in ((-1, 256), (129, 256), (0, 64), (0, (1 << 31) - 1)):
        assert lib.nmarl_policy_step_p(ctypes.byref(m), ctypes.byref(_fwd(128, env0, B_total)), None) != 0
        msg = lib.nmarl_last_error().decode()
        assert 'B_total' in msg or 'lane' in msg, msg


def test_env_resets_refuse_a_negative_env0():
    cfg, lib = L.CaccCfg(), L.lib()
    cfg.n_agent, cfg.platoon_len = 8, 8
    assert lib.nmarl_cacc_reset_shard(ctypes.byref(cfg), 4, *([None] * 2), 0, *([None] * 8), 8, None, 4, None, -1) != 0
    assert 'env0' in lib.nmarl_last_error().decode()


# ---- records from gathered per-rank arrays ---------------------------------------------------------------------------
def _as_ranks(monkeypatch, world, fn):
    """Run fn(rank) for every rank of `world` with gather_to_root standing in for the collective: ranks 1.. hand
    their object over, rank 0 receives all of them.  -> rank 0's result."""
    sent = {}

    def gather(obj, rank):
        sent[rank] = obj
        return [sent[r] for r in range(world)] if rank == 0 else None

    for rank in list(range(1, world)) + [0]:
        monkeypatch.setattr(D, 'gather_to_root', lambda obj, r=rank: gather(obj, r))
        out = fn(rank)
        assert (out is None) == (rank != 0)
    return out


class _Env:
    agent = 'ma2c_nc'
    par_stats = CACCEnv.par_stats

    def __init__(self, tab, lo, hi, total):
        self.tab, self.lo, self.hi = tab, lo, hi
        self.n_env, self.n_env_total, self.env_par = hi - lo, total, True

    def par_table(self):
        return {k: v[self.lo:self.hi].copy() for k, v in self.tab.items()}


def _vec(grew, env):
    vt = U.VecTrainer.__new__(U.VecTrainer)
    vt.env, vt.data, vt.par_data = env, [], []
    vt.engine = types.SimpleNamespace(grew_buf=grew, T_cur=grew.shape[0])
    return vt


@pytest.mark.parametrize('world', [2, 3, 8])
def test_train_records_from_gathered_shards_equal_the_one_process_records(world, monkeypatch):
    rs = np.random.RandomState(world)
    T, total = 60, 24 * world
    grew = torch.from_numpy(rs.standard_normal((T, total)) * 300 - 900)
    tab = {f: rs.uniform(1, 30, total) for f in L.ENV_PAR_FIELDS}
    tab['scenario'] = rs.randint(0, 2, total).astype(np.int32)
    one = _vec(grew, _Env(tab, 0, total, total))
    one.log_rewards(600)
    per = total // world

    def rank(r):
        vt = _vec(grew[:, r * per:(r + 1) * per].clone(), _Env(tab, r * per, (r + 1) * per, total))
        return None if vt.log_rewards(600) is None else vt

    many = _as_ranks(monkeypatch, world, rank)
    assert repr(many.data) == repr(one.data) and repr(many.par_data) == repr(one.par_data)


@pytest.mark.parametrize('world', [2, 3, 8])
def test_test_rewards_from_gathered_seed_shards_equal_the_one_process_rewards(world, monkeypatch):
    rs = np.random.RandomState(world)
    seeds = list(range(10000, 10000 + 10 * 11, 10))
    episodes = {s: rs.standard_normal(1 + rs.randint(5, 40)) * 200 - 700 for s in seeds}

    def make(rank, w):
        ev = U.BatchedEvaluator.__new__(U.BatchedEvaluator)
        ev.world, ev.rank = w, rank
        ev.episodes = lambda ss: ((k, len(episodes[s]) - 1, None, episodes[s], None) for k, s in enumerate(ss))
        return ev

    one = make(0, 1).test_rewards(seeds)
    many = _as_ranks(monkeypatch, world, lambda r: make(r, world).test_rewards(seeds))
    assert np.asarray(one).tobytes() == np.asarray(many).tobytes()


# ---- launching: nothing outlives a timed-out torchrun ------------------------------------------------------------------
_STUBBORN = """
import os, signal, sys, time
signal.signal(signal.SIGTERM, signal.SIG_IGN)          # a rank that does not stop when asked
open(os.path.join(sys.argv[1], 'pid%s' % os.environ['RANK']), 'w').write(str(os.getpid()))
time.sleep(600)
"""


def test_run_bounded_stops_torchrun_and_every_worker_on_timeout(tmp_path):
    import os
    import sys
    import time
    script = tmp_path / 'stubborn.py'
    script.write_text(_STUBBORN)
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--standalone', '--nproc-per-node', '2', str(script),
           str(tmp_path)]
    t0 = time.time()
    rc, _ = D.run_bounded(cmd, timeout=40, grace=5)                 # 40 s: ample for the workers to start
    assert rc is None and time.time() - t0 < 120
    pids = [int((tmp_path / ('pid%d' % r)).read_text()) for r in range(2)]        # the workers had started
    for pid in pids:
        assert not os.path.exists('/proc/%d' % pid) or open('/proc/%d/stat' % pid).read().split(')')[1].split()[0] == 'Z'
