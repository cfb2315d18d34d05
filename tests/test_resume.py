"""CPU: the files and checks of a resumable batched training run (TRAIN_CONFIG.checkpoint_interval, main.py train
--resume): the configuration comparison, every refusal, snapshot selection, retention, atomic writes, that `load`
still picks the newest checkpoint, and the global-env-order slicing that lets a snapshot of W processes restore
into W' processes."""
import configparser
import os
import types

import pytest
import torch

import main
from deeprl_network_b200 import dist as D
from deeprl_network_b200 import resume as R
from deeprl_network_b200.agents import models as agent_models
from helpers import ROOT


def _ini_text(**over):
    cp = configparser.ConfigParser()
    cp.read(os.path.join(ROOT, 'config', 'config_ma2c_nc_catchup.ini'))
    for key, v in over.items():
        sec, k = key.split('__')
        cp[sec][k] = str(v)
    from io import StringIO
    s = StringIO()
    cp.write(s)
    return s.getvalue()


def _write_ini(tmp_path, **over):
    path = tmp_path / 'exp.ini'
    path.write_text(_ini_text(**over))
    return str(path)


# ---- configuration comparison ----------------------------------------------------------------------------------------
def test_only_total_step_may_differ():
    base = _ini_text(ENV_CONFIG__n_env=8)
    assert R.config_difference(base, _ini_text(ENV_CONFIG__n_env=8, TRAIN_CONFIG__total_step=2e6)) is None
    assert R.config_difference(base, base) is None
    assert R.config_difference(base, _ini_text(ENV_CONFIG__n_env=8, MODEL_CONFIG__lr_init=1e-3))[0] == \
        'MODEL_CONFIG.lr_init'
    assert R.config_difference(base, _ini_text(ENV_CONFIG__n_env=8, ENV_CONFIG__slowdown_prob=0.5))[0] == \
        'ENV_CONFIG.slowdown_prob'                                                     # a key only one side has
    snap = dict(config=base, n_env=8)
    R.check_resumable(snap, _ini_text(ENV_CONFIG__n_env=8, TRAIN_CONFIG__total_step=5e6), 8)
    with pytest.raises(ValueError, match='TRAIN_CONFIG.log_interval'):
        R.check_resumable(snap, _ini_text(ENV_CONFIG__n_env=8, TRAIN_CONFIG__log_interval=7), 8)
    with pytest.raises(ValueError, match='16 envs in total.*n_env is 8'):
        R.check_resumable(dict(config=base, n_env=16), base, 8)


# ---- refusals of main.py train, before any GPU or collective call ---------------------------------------------------------
def _snapshot_file(base, step, config_text, n_env):
    os.makedirs(os.path.join(base, 'model'), exist_ok=True)
    R.save_snapshot(os.path.join(base, 'model'), step, {}, config_text, n_env)


def _train(base, ini, resume=True):
    argv = ['--base-dir', str(base), 'train', '--config-dir', ini] + (['--resume'] if resume else [])
    main.train(main.parse_args(argv))


def test_refusals(tmp_path, monkeypatch):
    for k in ('WORLD_SIZE', 'RANK', 'LOCAL_RANK'):
        monkeypatch.delenv(k, raising=False)
    base = tmp_path / 'run'
    with pytest.raises(ValueError, match='n_env > 1'):
        _train(base, _write_ini(tmp_path, ENV_CONFIG__n_env=1))
    with pytest.raises(ValueError, match='n_env > 1'):
        _train(base, _write_ini(tmp_path, ENV_CONFIG__n_env=1, TRAIN_CONFIG__checkpoint_interval=6000), resume=False)
    with pytest.raises(ValueError, match='no snapshot'):
        _train(base, _write_ini(tmp_path, ENV_CONFIG__n_env=8))
    _snapshot_file(str(base), 480, _ini_text(ENV_CONFIG__n_env=16), 16)
    with pytest.raises(ValueError, match='16 envs in total'):
        _train(base, _write_ini(tmp_path, ENV_CONFIG__n_env=8))
    with pytest.raises(ValueError, match='MODEL_CONFIG.num_fc'):
        _train(base, _write_ini(tmp_path, ENV_CONFIG__n_env=16, MODEL_CONFIG__num_fc=32))
    monkeypatch.setenv('WORLD_SIZE', '3')
    monkeypatch.setenv('RANK', '1')
    with pytest.raises(ValueError, match='multiple of the 3 processes'):
        _train(base, _write_ini(tmp_path, ENV_CONFIG__n_env=16))
    assert not os.path.exists(base / 'data') and not os.path.exists(base / 'log')     # nothing was started


class _Started(Exception):
    pass


def test_resume_from_the_ini_stored_in_data(tmp_path, monkeypatch):
    """--config-dir D/data/exp.ini --resume: data/ keeps that file (the run's configuration), and only it."""
    for k in ('WORLD_SIZE', 'RANK', 'LOCAL_RANK'):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setattr(main.U, 'init_log', lambda d: None)

    def started(*a, **k):                 # the .ini handling is done; the env would need a GPU
        raise _Started
    monkeypatch.setattr(main, 'init_env', started)
    base = tmp_path / 'run'
    text = _ini_text(ENV_CONFIG__n_env=16)
    os.makedirs(base / 'data')
    (base / 'data' / 'exp.ini').write_text(text)
    (base / 'data' / 'older.ini').write_text(text)
    _snapshot_file(str(base), 480, text, 16)
    with pytest.raises(_Started):
        _train(base, str(base / 'data' / 'exp.ini'))
    assert sorted(os.listdir(base / 'data')) == ['exp.ini']
    assert (base / 'data' / 'exp.ini').read_text() == text
    # a longer run from a config elsewhere replaces it
    longer = _write_ini(tmp_path, ENV_CONFIG__n_env=16, TRAIN_CONFIG__total_step=5e6)
    with pytest.raises(_Started):
        _train(base, longer)
    assert sorted(os.listdir(base / 'data')) == ['exp.ini']
    assert (base / 'data' / 'exp.ini').read_text() == open(longer).read()


class _Loop:
    """Stand-in for VecTrainer: an update counter and the env steps of the records it was asked to take."""

    def __init__(self, env, model, graph=True):
        self.n_update, self.data, self.graph = 0, [], None

    def start(self):
        pass

    def restore(self, snap):
        self.n_update, self.data = snap['n_update'], list(snap['data'])

    def update(self):
        self.n_update += 1

    def log_rewards(self, step, writer=None):
        self.data.append(step)
        return 0.0

    def snapshot(self):
        return dict(n_update=self.n_update, data=list(self.data))

    def write_csv(self, path):
        _Loop.written = list(self.data)


def _batched(total, resume=None):
    """_train_batched with 10 env steps per update, a record every 2 updates and a checkpoint every 3 ->
    ({env steps: snapshot}, records written)."""
    snaps = {}
    env, model = types.SimpleNamespace(n_env_total=2, test_seeds=[]), types.SimpleNamespace(n_step=5)
    main._train_batched(env, model, total, 20, output_path='unused', resume=resume, checkpoint_interval=30,
                        checkpoint=lambda run, step: snaps.__setitem__(step, run))
    return snaps, _Loop.written


def test_records_of_a_resumed_run_are_the_uninterrupted_runs(monkeypatch):
    """A first run that stops off the log cadence (update 3 of a record every 2) logs its last update, but the
    snapshot taken there holds only the records on the cadence, so a longer resumed run writes what one run writes."""
    monkeypatch.setattr(main.U, 'VecTrainer', _Loop)
    _, whole = _batched(60)
    assert whole == [20, 40, 60]
    snaps, first = _batched(30)
    assert first == [20, 30] and snaps[30]['loop']['data'] == [20]
    _, resumed = _batched(60, resume=snaps[30])
    assert resumed == whole


# ---- files ------------------------------------------------------------------------------------------------------------
def _touch(d, *names):
    for n in names:
        open(os.path.join(d, n), 'wb').close()


def test_newest_snapshot_ignores_other_and_temporary_files(tmp_path):
    d = str(tmp_path)
    assert R.newest_snapshot(d) is None and R.newest_snapshot(os.path.join(d, 'none')) is None
    _touch(d, 'resume-900.pt', 'resume-12000.pt', 'resume-3000.pt', '.resume-99999.pt.17.tmp', 'resume-50000.pt.tmp',
           'resume-x.pt', 'checkpoint-70000.pt', 'resume-60000.pt~')
    assert R.newest_snapshot(d) == os.path.join(d, 'resume-12000.pt')


def test_atomic_save_leaves_only_the_final_name(tmp_path):
    d = str(tmp_path)
    R.save_snapshot(d, 120, {'x': torch.arange(3)}, '[A]\nk = v\n', 4)
    assert os.listdir(d) == ['resume-120.pt']
    snap = R.load_snapshot(R.newest_snapshot(d))
    assert snap['step'] == 120 and snap['n_env'] == 4 and torch.equal(snap['run']['x'], torch.arange(3))


def test_load_picks_the_newest_checkpoint_beside_resume_files(tmp_path):
    d = str(tmp_path) + '/'
    stub = types.SimpleNamespace(engine=types.SimpleNamespace(
        params=torch.zeros(3), ms=torch.zeros(3), repack=lambda: None, _refresh_msg=lambda: None))
    for step in (100, 300, 200):
        torch.save({'params': torch.full((3,), float(step)), 'ms': torch.ones(3)}, d + 'checkpoint-%d.pt' % step)
    for step in (400, 500):
        R.save_snapshot(d, step, {}, '', 4)
    _touch(d, '.checkpoint-900.pt.5.tmp')
    assert agent_models.IA2C.load(stub, d)
    assert torch.equal(stub.engine.params, torch.full((3,), 300.0))


def test_retention_keeps_the_newest_five_of_each(tmp_path):
    d = str(tmp_path)
    steps = [60, 120, 180, 240, 300, 360, 420, 1200]
    _touch(d, *['checkpoint-%d.pt' % s for s in steps], *['resume-%d.pt' % s for s in steps[1:]], 'notes.txt')
    R.prune(d)
    keep = steps[-5:]
    assert sorted(os.listdir(d)) == sorted(['checkpoint-%d.pt' % s for s in keep] + ['resume-%d.pt' % s for s in keep]
                                           + ['notes.txt'])


# ---- global env order across process counts ---------------------------------------------------------------------------------
@pytest.mark.parametrize('w_from,w_to', [(2, 1), (1, 2), (4, 2), (2, 4), (8, 1)])
def test_slices_move_between_process_counts(w_from, w_to):
    n = 8
    glob = dict(state=torch.arange(3 * n * 5).reshape(3, n, 5), done=torch.arange(n) * 10,
                par=torch.arange(n * 2).reshape(n, 2))
    axes = dict(state=1, done=0, par=0)
    # the ranks of the writing run each hold their shard; rank 0 concatenates them in rank order
    parts = [D.take_envs(glob, axes, *D.env_shard(n, w_from, r)) for r in range(w_from)]
    gathered = D.concat_envs(parts, axes)
    for k in glob:
        assert torch.equal(gathered[k], glob[k])
    # every rank of the resuming run takes its own envs out of the global order
    for r in range(w_to):
        env0, per = D.env_shard(n, w_to, r)
        mine = D.take_envs(gathered, axes, env0, per)
        assert torch.equal(mine['state'], glob['state'][:, env0:env0 + per])
        assert torch.equal(mine['done'], glob['done'][env0:env0 + per])
        assert torch.equal(mine['par'], glob['par'][env0:env0 + per])
    with pytest.raises(ValueError, match='not the envs 6 .. 9'):
        D.take_envs(gathered, axes, 6, 4)
