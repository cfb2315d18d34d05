"""Experiment plumbing and the two training loops.

Drop-in surface (names, arguments and observable behaviour of the reference's utils.py:11-60, 70-97, 100-254,
311-336): ``Counter``, ``Trainer`` with ``explore`` / ``perform`` / ``run``, ``Tester``, ``Evaluator`` and the
directory / logging helpers.  The single-environment ``Trainer`` reproduces the reference loop call for call --
tests/test_trainer_flow.py replays traces recorded from the reference's own Trainer bit for bit -- including
its quirks (SURVEY 8a): Q1 the value call follows the policy call on the already advanced recurrent state, Q2 the
bootstrap at a non-terminal batch end is one more policy + value call, Q4 the reward that gets logged for CACC is
that of a greedy test episode run after every training episode, Q5 only training steps are counted.

``VecTrainer`` is the batched loop this package adds (n_env parallel episodes, everything device resident,
optionally one process per GPU with one NCCL gradient all-reduce per update).  ``BatchedEvaluator`` runs the greedy
test episodes of many seeds at once on the device and writes what ``Evaluator`` writes, byte for byte.
"""
import logging
import pathlib
import shutil
import time

import numpy as np
import torch

from . import _lib as L
from . import dist as D
from .agents.engine import PolicyEngine
from .envs.cacc_env import CACCEnv, control_record, env_par_keys, nominal_config, traffic_frame, write_records
from .layout import ModelLayout

_TEST_MODES = {'no_test': (False, False), 'in_train_test': (True, False),
               'after_train_test': (False, True), 'all_test': (True, True)}


# ---- directories / logging ---------------------------------------------------------------------------------------
def check_dir(cur_dir):
    return pathlib.Path(cur_dir).exists()


def copy_file(src_dir, tar_dir):
    shutil.copy(src_dir, tar_dir)


def find_file(cur_dir, suffix='.ini'):
    root = pathlib.Path(cur_dir)
    hits = sorted(f for f in root.iterdir() if f.name.endswith(suffix)) if root.is_dir() else []
    if hits:
        return '%s/%s' % (cur_dir, hits[0].name)
    logging.error('Cannot find %s file' % suffix)
    return None


def init_dir(base_dir, pathes=('log', 'data', 'model')):
    """-> {'log': '<base>/log/', ...}; creates what is missing."""
    out = {}
    for sub in pathes:
        d = pathlib.Path(base_dir) / sub
        d.mkdir(parents=True, exist_ok=True)
        out[sub] = '%s/%s/' % (base_dir, sub)
    return out


def init_log(log_dir):
    stamp = int(time.time())
    logging.basicConfig(format='%(asctime)s [%(levelname)s] %(message)s', level=logging.INFO,
                        handlers=[logging.FileHandler('%s/%d.log' % (log_dir, stamp)), logging.StreamHandler()])


def init_test_flag(test_mode):
    return _TEST_MODES.get(test_mode, (False, False))


def make_summary_writer(log_dir):
    """TensorBoard event writer (stands in for tf.summary.FileWriter); None when tensorboard is absent."""
    try:
        from torch.utils.tensorboard import SummaryWriter
        return SummaryWriter(log_dir)
    except Exception:  # pragma: no cover
        logging.warning('tensorboard not available: scalar summaries disabled')
        return None


class Counter:
    """Global step bookkeeping: counts training steps only; test / log cadence; stop condition."""

    def __init__(self, total_step, test_step, log_step):
        self.total_step, self.test_step, self.log_step = total_step, test_step, log_step
        self.cur_step = self.cur_test_step = 0
        self.stop = False

    def next(self):
        self.cur_step += 1
        return self.cur_step

    def should_test(self):
        due = self.cur_step - self.cur_test_step >= self.test_step
        if due:
            self.cur_test_step = self.cur_step
        return due

    def should_log(self):
        return self.cur_step % self.log_step == 0

    def should_stop(self):
        return self.stop or self.cur_step >= self.total_step


# ---- the single-environment loop -----------------------------------------------------------------------------------
class _AgentPort:
    """The two call conventions of the agent classes behind one face.  MA2C-style agents take the whole
    fingerprint matrix with every call and the joint action for the value; IA2C-style agents take nothing extra
    for the policy and, per agent, its neighbours' actions for the value.  ``aux`` is whatever the last call used
    and is what ``add_transition`` stores next to the observation."""

    def __init__(self, env, model):
        self.env, self.model = env, model
        self.joint = env.agent.startswith('ma2c')
        self.aux = None

    def policy(self, ob, done):
        if not self.joint:
            return self.model.forward(ob, done)
        self.aux = self.env.get_fingerprint()
        return self.model.forward(ob, done, self.aux)

    def value(self, ob, done, action):
        if self.joint:
            return self.model.forward(ob, done, self.aux, np.array(action), 'v')
        self.aux = self.env.get_neighbor_action(action)
        return self.model.forward(ob, done, self.aux, 'v')

    def store(self, ob, action, reward, value, done):
        self.model.add_transition(ob, self.aux, action, reward, value, done)


class Trainer:
    """One environment, one episode at a time (the reference's protocol).  ``uniform_fn`` optionally supplies the
    uniform behind each sampled action (tests feed the CUDA path and the oracle the same stream); by default
    actions come from ``np.random.choice`` like in the reference."""

    def __init__(self, env, model, global_counter, summary_writer, output_path=None, uniform_fn=None):
        if getattr(env, 'env_par', None) is not None:
            raise ValueError('per-env scenario parameters (ENV_CONFIG *_range / slowdown_prob) need batched training '
                             '(VecTrainer, n_env > 1)')
        self.env, self.model, self.global_counter = env, model, global_counter
        self.summary_writer, self.output_path, self.uniform_fn = summary_writer, output_path, uniform_fn
        self.agent = env.agent
        self.sess = getattr(model, 'sess', None)
        self.n_step = model.n_step
        if env.T % self.n_step:
            raise AssertionError('episode length %d is not a multiple of the batch size %d' % (env.T, self.n_step))
        self.cur_step = 0
        self.data = []
        self.episode_rewards = []
        self.env.train_mode = True
        self._port = _AgentPort(env, model)

    # -- action selection --
    def _draw(self, pi):
        if self.uniform_fn is None:
            return np.random.choice(np.arange(len(pi)), p=pi)
        cdf = np.cumsum(np.asarray(pi, dtype=np.float64))
        return int(np.searchsorted(cdf / cdf[-1], self.uniform_fn(), side='right'))

    def _decide(self, ob, done, greedy=False):
        policy = self._port.policy(ob, done)
        pick = np.argmax if greedy else self._draw
        return policy, np.array([pick(pi) for pi in policy])

    # -- logging --
    def _add_summary(self, reward, global_step, is_train=True):
        if self.summary_writer is not None:
            self.summary_writer.add_scalar('train_reward' if is_train else 'test_reward', reward, global_step)

    def _log_episode(self, global_step, mean_reward, std_reward):
        self.data.append(dict(agent=self.agent, step=global_step, test_id=-1, avg_reward=mean_reward,
                              std_reward=std_reward))
        self._add_summary(mean_reward, global_step)
        if self.summary_writer is not None:
            self.summary_writer.flush()

    # -- one batch of at most n_step transitions + its bootstrap target --
    def explore(self, prev_ob, prev_done):
        ob, done, port = prev_ob, prev_done, self._port
        for _ in range(self.n_step):
            policy, action = self._decide(ob, done)
            value = port.value(ob, done, action)                  # Q1: evaluated after the policy call
            self.env.update_fingerprint(policy)
            nxt, reward, done, global_reward = self.env.step(action)
            self.episode_rewards.append(global_reward)
            step = self.global_counter.next()
            self.cur_step += 1
            port.store(ob, action, reward, value, done)
            if self.global_counter.should_log():
                logging.info('Training: global step %d, episode step %d, ob: %s, a: %s, pi: %s, r: %.2f, '
                             'train r: %.2f, done: %r' % (step, self.cur_step, ob, action, policy, global_reward,
                                                          np.mean(reward), done))
            if done:                                              # CACC episodes may end inside a batch
                return ob, done, np.zeros(self.model.n_agent)
            ob = nxt
        _, action = self._decide(ob, done)                        # Q2: the bootstrap is a full policy + value call
        return ob, done, port.value(ob, done, action)

    # -- one evaluation episode --
    def perform(self, test_ind, gui=False):
        ob, done = self.env.reset(gui=gui, test_ind=test_ind), True      # done=True clears the recurrent state
        self.model.reset()
        greedy = not self.env.name.startswith('atsc')                    # CACC is evaluated with the arg-max policy
        rewards = []
        while True:
            policy, action = self._decide(ob, done, greedy=greedy)
            self.env.update_fingerprint(policy)
            ob, _, done, global_reward = self.env.step(action)
            rewards.append(global_reward)
            if done:
                rewards = np.array(rewards)
                return np.mean(rewards), np.std(rewards)

    def _train_episode(self):
        ob, done = self.env.reset(), True
        self.model.reset()
        self.cur_step, self.episode_rewards = 0, []
        while True:
            ob, done, R = self.explore(ob, done)
            step = self.global_counter.cur_step
            self.model.backward(R, self.env.T - self.cur_step, self.summary_writer, step)
            if done:
                self.env.terminate()
                return step

    def run(self, max_episodes=None):
        episodes = 0
        while not self.global_counter.should_stop() and (max_episodes is None or episodes < max_episodes):
            step = self._train_episode()
            rewards = np.array(self.episode_rewards)
            mean_reward, std_reward = np.mean(rewards), np.std(rewards)
            if not self.env.name.startswith('atsc'):              # Q4: a greedy episode provides the logged reward
                self.env.train_mode = False
                mean_reward, std_reward = self.perform(-1)
                self.env.train_mode = True
            self._log_episode(step, mean_reward, std_reward)
            episodes += 1
        if self.output_path is not None:
            import pandas as pd
            pd.DataFrame(self.data).to_csv(self.output_path + 'train_reward.csv')


class Tester(Trainer):
    """Present in the reference's import list but never run by its main.py (SURVEY row 11); kept so that the
    import keeps working."""

    def __init__(self, env, model, global_counter, summary_writer, output_path):
        super().__init__(env, model, global_counter, summary_writer, output_path=output_path)
        self.env.train_mode = False
        self.test_num = env.test_num


class Evaluator(Tester):
    """Runs every test seed of the environment once with the loaded model and writes the episode records."""

    def __init__(self, env, model, output_path, gui=False):
        self.env, self.model, self.output_path, self.gui = env, model, output_path, gui
        self.agent = env.agent
        self.env.train_mode = False
        self.test_num = env.test_num
        self.uniform_fn = None
        self._port = _AgentPort(env, model)

    def run(self):
        self.env.cur_episode = 0
        self.env.init_data(not self.gui, False, self.output_path)
        for test_ind in range(self.test_num):
            reward, _ = self.perform(test_ind, gui=self.gui)
            self.env.terminate()
            logging.info('test %i, avg reward %.2f' % (test_ind, reward))
            self.env.collect_tripinfo()
        self.env.output_data()


class VecTrainer:
    """Batched training loop: n_env parallel episodes advance in lock-step on the device.

    Per update: ``rollout`` (n_step x [p-call, v-call, env step] + bootstrap) -> returns ->
    training forward/BPTT/wgrad -> [all-reduce] -> clip + RMSProp, then per-env auto-reset of the
    environments whose episode ended (model.reset() + env.reset() of the reference, per env).
    With ``graph=True`` one update is captured once into a CUDA graph and replayed.

    When the env is one shard of a run over several processes (env.n_env_total > env.n_env), the records gather
    every rank's envs to rank 0 in global env order and are computed there on what one process would hold; the other
    ranks record nothing.
    """

    def __init__(self, env, model, graph=True, sample='philox'):
        self.env, self.model, self.engine = env, model, model.engine
        assert env.n_env == model.n_env
        self.sample = sample
        self.use_graph = graph
        self.graph = None
        self.n_update = 0
        self.env.train_mode = True
        # Episodes end (env `done`) only at multiples of the env's batch_size and at T: the per-env auto-reset below
        # looks at the done flag of the LAST step of an update only, so updates must tile the episode exactly
        # (the reference's Trainer has the same requirement implicitly, utils.py:129-197).
        if env.T % model.n_step or env.batch_size % model.n_step:
            raise AssertionError('VecTrainer: episode length %d / env batch_size %d are not multiples of the update '
                                 'length %d' % (env.T, env.batch_size, model.n_step))
        self.data = []                     # one record per update (train_reward.csv of the batched loop)
        self.par_data = []                 # with per-env scenario parameters: env_par.csv, one row per log record

    def start(self):
        self._seed = self.env.seed
        self.env.reset_device(u01=None, philox_seed=self._seed)
        self.engine.reset_states()
        self.engine.begin_episode(self.env)

    def _one_update(self, uniforms=None):
        e, env = self.engine, self.env
        e.rollout(env, sample=self.sample, uniforms=uniforms)
        e.update(self._lr)
        # episode boundaries: envs whose last step returned done restart (per-env model.reset/env.reset)
        done = e.done_buf[e.T_cur]
        e.roll_buffers()
        e.reset_states(mask=done)
        env.reset_device(u01=None, mask=done, obs_out=e.obs_buf[0], fp_out=e.fp_buf[0], philox_seed=self._seed)
        e.normalize_cur()

    def update(self, uniforms=None):
        e = self.engine
        # the schedule counts ENVIRONMENT steps (main.py's total_step): one update consumes n_step steps of every
        # env on every rank, so a linear lr_decay reaches lr_min at total_step whatever n_env / world size is
        lr = self.model.lr_scheduler.get(self.model.n_step * self.env.n_env * e.world)
        e.lr_dev.fill_(float(lr))
        self._lr = e.lr_dev
        if not self.use_graph:
            self._one_update(uniforms)
        else:
            if self.graph is None:
                self._static_uniforms = uniforms
                # warm-up outside capture (sets kernel attributes, allocates training buffers)
                self._one_update(uniforms)
                torch.cuda.synchronize()
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph):
                    self._one_update(self._static_uniforms)
                self.n_update += 1
                return
            self.graph.replay()
        self.n_update += 1

    def mean_reward(self):
        """Mean per-step global reward of the last batch (host sync)."""
        return float(self.engine.grew_buf[:self.engine.T_cur].mean().item())

    def log_rewards(self, global_step, summary_writer=None):
        """One `train_reward.csv` record (same columns as Trainer._log_episode): mean / std of the per-step global
        reward over the last batch of every env.  Unlike the one-env Trainer (quirk Q4) no greedy test episode is
        interleaved: these are the TRAINING rewards.  Host sync.  Returns the mean (None on ranks other than 0 of a
        sharded run)."""
        g = self.engine.grew_buf[:self.engine.T_cur]
        tab = self.env.par_table() if getattr(self.env, 'env_par', None) is not None else None
        if self.env.n_env_total != self.env.n_env:
            parts = D.gather_to_root((g.cpu().numpy(), tab))
            if parts is None:
                return None
            g = torch.from_numpy(np.concatenate([p[0] for p in parts], axis=1)).to(g.device)
            if tab is not None:
                tab = {k: np.concatenate([p[1][k] for p in parts]) for k in tab}
        mean, std = float(g.mean().item()), float(g.std(unbiased=False).item())
        self.data.append(dict(agent=self.env.agent, step=int(global_step), test_id=-1, avg_reward=mean, std_reward=std))
        if tab is not None:
            self.par_data.append(dict(step=int(global_step), **self.env.par_stats(tab)))
        if summary_writer is not None:
            summary_writer.add_scalar('train_reward', mean, int(global_step))
        return mean

    def snapshot(self):
        """The run state between two updates, in a layout that depends neither on the process count nor on the kernel
        path: the engine's and the env's (per-env tensors in global env order, gathered from every rank), the update
        count, the env reset seed, the schedule position and the records behind train_reward.csv / env_par.csv.  Every
        rank calls it (it checks that the Philox state agrees and gathers); rank 0 gets the snapshot, the others None."""
        D.check_replicas({'Philox state (engine.rng)': self.engine.rng})
        eng, env = self.engine.snapshot(), self.env.snapshot()
        parts = D.gather_to_root((eng['envs'], env['envs']))
        if parts is None:
            return None
        eng['envs'] = D.concat_envs([p[0] for p in parts], eng['env_axis'])
        env['envs'] = D.concat_envs([p[1] for p in parts], env['env_axis'])
        return dict(engine=eng, env=env, n_update=self.n_update, seed=int(self._seed),
                    schedule_n=self.model.lr_scheduler.n,data=plain_records(self.data),
                    par_data=plain_records(self.par_data))

    def restore(self, snap):
        """Put a snapshot back in place: after start() and before the first update, so that the CUDA graph the first
        update captures reads the restored tensors.  Each rank takes its own envs of the snapshot's global order."""
        if self.graph is not None or self.n_update:
            raise RuntimeError('VecTrainer.restore runs after start() and before the first update')
        self.engine.restore(snap['engine'])
        self.env.restore(snap['env'])
        self.n_update, self._seed = int(snap['n_update']), int(snap['seed'])
        self.model.lr_scheduler.n = snap['schedule_n']
        self.data, self.par_data = list(snap['data']), list(snap['par_data'])

    def write_csv(self, output_path):
        """train_reward.csv and, with per-env scenario parameters, env_par.csv: per log record the mean / min / max over
        the batch of every drawn field (the table as it stands at the record: the parameters of the running episodes)."""
        import pandas as pd
        pd.DataFrame(self.data).to_csv(output_path + 'train_reward.csv')
        if self.par_data:
            pd.DataFrame(self.par_data).to_csv(output_path + 'env_par.csv')


class BatchedEvaluator:
    """Greedy test episodes of many seeds in one pass on the device: what ``Evaluator`` does one seed at a time.

    Env b of a pass starts from test seed b with the host draws of ``CACCEnv.reset(test_ind=b)``; every step is one
    greedy p-call (pi goes straight into the next fingerprint slot), one test-mode env step and one
    ``nmarl_eval_record`` launch, with no host round trip until the pass ends.  The model is a second engine over
    the trained parameter tensor itself: no weights are copied, and the trained model's states, RNG and buffers are
    not touched.

    It always runs the FP32-FFMA kernels.  Their per-row arithmetic does not depend on the number of envs and the env
    step is per env, so every action, and therefore every file, equals the one-env ``Evaluator``'s bit for bit; the
    tensor-core kernels round differently and would flip near-tie arg-maxes.

    Seeds go through in passes of at most ``max_env`` envs whose records fit in ``record_bytes`` of device memory
    (DESIGN §4.7).  With ``graph`` the steps of a pass are captured into a CUDA graph on the second pass of a size
    and replayed from then on.

    Evaluation always runs the config's nominal scenario parameters: per-env parameter keys (``*_range``,
    ``slowdown_prob``) of a training config are ignored here, so test rewards stay comparable across runs.

    In a run over several processes (``world`` > 1) ``test_rewards`` runs rank ``rank``'s contiguous part of the
    seeds and reduces every rank's episodes on rank 0, in seed order.
    """

    def __init__(self, env_config, model, output_path=None, max_env=4096, record_bytes=2 ** 31, graph=True, world=1,
                 rank=0):
        if env_par_keys(env_config):
            env_config = nominal_config(env_config)
        self.config, self.model, self.output_path = env_config, model, output_path
        self.max_env, self.record_bytes, self.use_graph = int(max_env), int(record_bytes), graph
        self.layout = self._eval_layout(model.layout)
        self.agent = env_config.get('agent')
        self._runners = {}
        self.data = []                     # test_reward.csv records (log_test)
        self.world, self.rank = int(world), int(rank)

    @staticmethod
    def _eval_layout(lay):
        if getattr(lay, 'hetero', False):
            raise ValueError('batched evaluation runs homogeneous agents (the CACC platoons have them)')
        if lay.variant == 'ia2c' and lay.obs_mode != 'gather':
            # device rollouts gather the neighbours' observation rows in the kernel; the one-env model reads the
            # caller's concatenation.  Both give the kernel the same input row and the same parameter layout.
            g = ModelLayout('ia2c', lay.n_s_ls, lay.n_a, lay.mask, n_h=lay.n_h, n_fc=lay.n_h, obs_mode='gather')
            assert g.entries == lay.entries and g.n_param == lay.n_param and g.kx_pad == lay.kx_pad
            return g
        return lay

    def chunk_size(self, n_seed):
        """Envs per pass: at most max_env, and records of at most record_bytes."""
        lay, T = self.layout, self._episode_len()
        per_env = (T + 1) * (lay.N * (4 + 3 * 8) + 8)
        return max(1, min(self.max_env, int(n_seed), self.record_bytes // per_env))

    def _episode_len(self):
        return int(self.config.getint('episode_length_sec') / self.config.getfloat('control_interval_sec'))

    def _runner(self, E):
        r = self._runners.get(E)
        if r is not None:
            return r
        src = self.model.engine
        env = CACCEnv(self.config, n_env=E, device=src.device)
        env.train_mode = False
        eng = PolicyEngine(self.layout, E, 1, dict(src.hp), device=src.device, use_tc=False, shared_params=src.params)
        T, N, dev = env.T, env.n_agent, src.device
        z = lambda *s, dtype=torch.float64: torch.zeros(*s, dtype=dtype, device=dev)
        r = dict(env=env, eng=eng, T=T, u01=z(*env.v_init.shape), alive=z(E, dtype=torch.int32),
                 steps=z(E, dtype=torch.int32), action=z(T + 1, E, N, dtype=torch.int32), reward=z(T + 1, E),
                 hs=z(T + 1, E, N), vs=z(T + 1, E, N), us=z(T + 1, E, N), graph=None, passes=0)
        self._runners[E] = r
        return r

    def _record(self, r, start, done=None):
        env, eng = r['env'], r['eng']
        L.check(L.lib().nmarl_eval_record(env.n_agent, env.n_env, r['T'], int(start), L.ptr(eng.act_buf[0]),
                                          L.ptr(env.greward_dev), L.ptr(done), L.ptr(env.hs), L.ptr(env.vs),
                                          L.ptr(env.us), L.ptr(r['alive']), L.ptr(r['steps']), L.ptr(r['action']),
                                          L.ptr(r['reward']), L.ptr(r['hs']), L.ptr(r['vs']), L.ptr(r['us']),
                                          L.stream()), 'nmarl_eval_record')

    def _steps(self, r):
        """The T greedy steps of a pass.  Slots 0 / 1 of the engine's buffers take turns as 'now' and 'next'."""
        env, eng = r['env'], r['eng']
        for t in range(r['T']):
            s, n = t & 1, 1 - (t & 1)
            eng.step_p(eng.obs_buf[s], eng.fp_buf[s], eng.done_buf[s], eng.fp_buf[n], eng.act_buf[0], L.SAMPLE_GREEDY)
            env.step_device(eng.act_buf[0], obs_out=eng.obs_buf[n], done_out=eng.done_buf[n])   # rewards: env's own
            self._record(r, False, eng.done_buf[n])

    def _pass(self, seeds):
        """One greedy episode per seed, all at once -> host arrays (steps [E], action [T+1,E,N], reward [T+1,E],
        hs / vs / us [T+1,E,N]); episode b holds slots 0..steps[b]."""
        r = self._runner(len(seeds))
        env, eng = r['env'], r['eng']
        u = np.empty(tuple(r['u01'].shape))
        for b, seed in enumerate(seeds):              # CACCEnv.reset(test_ind): np.random.seed, then one draw per platoon
            np.random.seed(seed)
            u[:, b] = [np.random.rand() for _ in range(u.shape[0])]
        r['u01'].copy_(torch.from_numpy(u))
        eng.cur = 0                                   # the graph was captured from slot 0
        eng.reset_states()
        env.reset_device(u01=r['u01'], obs_out=eng.obs_buf[0], fp_out=eng.fp_buf[0])
        eng.done_buf[0].fill_(1.0)
        self._record(r, True)
        if self.use_graph and r['graph'] is None and r['passes'] > 0:
            r['graph'] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(r['graph']):
                self._steps(r)
        if r['graph'] is not None:
            r['graph'].replay()
        else:
            self._steps(r)
        r['passes'] += 1
        return tuple(r[k].cpu().numpy() for k in ('steps', 'action', 'reward', 'hs', 'vs', 'us'))

    def episodes(self, seeds):
        """The greedy episode of every seed, in seed order, as split_episodes yields them."""
        rng = np.random.get_state()                   # the host draws in _pass must not move the caller's stream
        try:
            E = self.chunk_size(len(seeds))
            for c0 in range(0, len(seeds), E):
                yield from split_episodes(c0, *self._pass(seeds[c0:c0 + E]))
        finally:
            np.random.set_state(rng)

    def run(self, seeds):
        """main.py evaluate: the two record files and the log lines of Evaluator.run for these test seeds."""
        name = self.config.get('scenario').split('_')[1]
        write_episode_records(self.episodes(list(seeds)), self.output_path, name, self.agent,
                              self.config.getfloat('control_interval_sec'))

    def test_rewards(self, seeds):
        """mean / std of the per-step global rewards of one greedy episode per seed, all episodes together (None on
        ranks other than 0 of a run over several processes)."""
        mine = [reward[1:] for _, _, _, reward, _ in self.episodes(D.seed_shard(seeds, self.world, self.rank))]
        if self.world > 1:
            parts = D.gather_to_root(mine)
            if parts is None:
                return None
            mine = [r for part in parts for r in part]
        r = np.concatenate(mine)
        return np.mean(r), np.std(r)

    def log_test(self, global_step, seeds, summary_writer=None):
        """One test_reward.csv record (columns of train_reward.csv) and the TB scalar `test_reward`.  Returns the
        mean (None on ranks other than 0 of a run over several processes)."""
        out = self.test_rewards(seeds)
        if out is None:
            return None
        mean, std = out
        self.data.append(dict(agent=self.agent, step=int(global_step), test_id=-1, avg_reward=mean, std_reward=std))
        if summary_writer is not None:
            summary_writer.add_scalar('test_reward', mean, int(global_step))
        return mean

    def write_csv(self, output_path):
        import pandas as pd
        pd.DataFrame(self.data).to_csv(output_path + 'test_reward.csv')

    def snapshot(self):
        """The test_reward.csv records so far (a resumed run writes the file whole)."""
        return plain_records(self.data)

    def restore(self, records):
        self.data = list(records)


def plain_records(records):
    """Records with NumPy scalars turned into Python numbers, which a snapshot loads without unpickling code (and
    which pandas writes to CSV exactly like the NumPy scalars)."""
    return [{k: v.item() if isinstance(v, np.generic) else v for k, v in r.items()} for r in records]


def split_episodes(first, steps, action, reward, hs, vs, us):
    """Host copies of one recorder pass -> (seed index, S, action [S, N], reward [S + 1], tr [S + 1, 3, N]) per
    episode of S steps, in the layout CACCEnv keeps while it records (reward[0] = 0 and tr[0] is the reset state)."""
    for b in range(len(steps)):
        S = int(steps[b])
        tr = np.empty((S + 1, 3, hs.shape[2]))
        tr[:, 0], tr[:, 1], tr[:, 2] = hs[:S + 1, b], vs[:S + 1, b], us[:S + 1, b]
        yield first + b, S, action[1:S + 1, b], np.ascontiguousarray(reward[:S + 1, b]), tr


def write_episode_records(episodes, output_path, name, agent, dt):
    """What Evaluator.run writes for these episodes: one `test %i, avg reward %.2f` log line each and, unless
    output_path is None, <name>_<agent>_control.csv / _traffic.csv.  Episode k is numbered k + 1, as the one-env
    env counts its resets from 0."""
    control, traffic = [], []
    for k, S, action, reward, tr in episodes:
        if output_path is not None:
            control.extend(control_record(k + 1, t, dt, action[t - 1], reward[t]) for t in range(1, S + 1))
            traffic.append(traffic_frame(k + 1, tr, reward, dt))
        logging.info('test %i, avg reward %.2f' % (k, np.mean(reward[1:].copy())))
    if output_path is not None:
        write_records(output_path, name, agent, control, traffic)
