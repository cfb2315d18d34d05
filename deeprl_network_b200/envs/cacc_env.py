"""CACC platoon environment, vectorised over B parallel episodes on the GPU.

Host-side mirror of the reference ``CACCEnv`` (envs/cacc_env.py): same constructor argument
(the ``ENV_CONFIG`` section), same methods and attributes (SURVEY 8b), so ``Trainer`` /
``main.py`` drive it unchanged.  With ``n_env == 1`` every call has the reference semantics
(seed stepping, test-episode seeds, fingerprints, IA2C observation concatenation).  The state
lives in device memory as float64 [agent][env] arrays and is advanced by the ``nmarl_cacc_*``
kernels (csrc/env.cu); ``*_device`` methods expose the batched tensors without host copies.

New optional keys in ``ENV_CONFIG`` (everything else parses exactly like the reference):
  n_env        parallel episodes in total (default 1); a process of a sharded run holds n_env / world of them
  platoon_len  vehicles per platoon (default n_vehicle); < n_vehicle gives several independent
               platoons -- used only by the synthetic 5x5-grid configuration
  topology     'chain' (default) or 'grid' (row-major 4-neighbour grid, Manhattan distance)
Per-env scenario parameters (batched training only, n_env > 1; all absent by default -- see ``parse_env_par``):
  <key>_range  = lo, hi  for headway_target, speed_target, headway_st, headway_go, speed_max, accel_min, accel_max:
               each env draws its own value from U[lo, hi) whenever it resets
  slowdown_prob = p      each env runs slow-down with probability p, else catch-up (default: `scenario` for all)
"""
import configparser
import ctypes as C
import logging

import numpy as np
import torch

from .. import _lib as L
from .. import dist as D


def chain_masks(n):
    """Chain adjacency and |i-j| distances (envs/cacc_env.py:253-267)."""
    nb = np.zeros((n, n), dtype=int)
    idx = np.arange(n)
    nb[idx[1:], idx[:-1]] = 1
    nb[idx[:-1], idx[1:]] = 1
    return nb, np.abs(idx[:, None] - idx[None, :]).astype(int)


def grid_masks(side):
    """4-neighbour side x side grid in row-major order with Manhattan distances -- equals the
    large-grid adjacency/distance of envs/large_grid_env.py:58-105 (SURVEY 8d, cfg5)."""
    n = side * side
    r, c = np.divmod(np.arange(n), side)
    dist = (np.abs(r[:, None] - r[None, :]) + np.abs(c[:, None] - c[None, :])).astype(int)
    return (dist == 1).astype(int), dist


# ENV_CONFIG key -> field of the per-env parameter table (nmarl_cacc_env_par), in table order
PAR_KEYS = dict(zip(('headway_target', 'speed_target', 'headway_st', 'headway_go', 'speed_max', 'accel_min',
                     'accel_max'), L.ENV_PAR_FIELDS))
ENV_PAR_KEYS = tuple(k + '_range' for k in PAR_KEYS) + ('slowdown_prob',)


def env_par_keys(config):
    """The per-env parameter keys present in an ENV_CONFIG section."""
    return [k for k in ENV_PAR_KEYS if k in config]


def nominal_config(config):
    """A copy of an ENV_CONFIG section without the per-env parameter keys: every env runs the config's nominal
    values.  Evaluation uses it, so that test rewards stay comparable across runs."""
    cp = configparser.ConfigParser(interpolation=None)
    cp.read_dict({'ENV_CONFIG': {k: config.get(k, raw=True) for k in config if k not in ENV_PAR_KEYS}})
    return cp['ENV_CONFIG']


def parse_env_par(config, h_min=None):
    """ENV_CONFIG section -> the draw ranges of the per-env parameter table, or None when no key is present.

    Returns {'ranges': {field: (lo, hi)} for every field of L.ENV_PAR_FIELDS (a field without its key gets the
    point range of its nominal value), 'slowdown_prob': p or None}.  Raises ValueError, naming the key, unless
    lo <= hi for every range and every draw keeps headway_min < headway_st < headway_go, accel_min < 0 < accel_max,
    speed_target > 0 and headway_target > 0, and 0 <= slowdown_prob <= 1 (the checks nmarl_cacc_draw_par repeats)."""
    if not env_par_keys(config):
        return None
    h_min = config.getfloat('headway_min') if h_min is None else h_min
    ranges = {}
    for key, field in PAR_KEYS.items():
        if key + '_range' not in config:
            v = config.getfloat(key)
            ranges[field] = (v, v)
            continue
        txt = config.get(key + '_range')
        try:
            lo, hi = (float(x) for x in txt.split(','))
        except ValueError:
            raise ValueError('ENV_CONFIG.%s_range = %r: expected two numbers "lo, hi"' % (key, txt)) from None
        if not lo <= hi:
            raise ValueError('ENV_CONFIG.%s_range = %r: needs lo <= hi' % (key, txt))
        ranges[field] = (lo, hi)
    lo = {f: r[0] for f, r in ranges.items()}
    hi = {f: r[1] for f, r in ranges.items()}
    if not h_min < lo['h_s']:
        raise ValueError('headway_st (from %g) must exceed headway_min (%g) for every draw' % (lo['h_s'], h_min))
    if not hi['h_s'] < lo['h_g']:
        raise ValueError('headway_st (up to %g) must stay below headway_go (from %g) for every draw'
                         % (hi['h_s'], lo['h_g']))
    if not hi['u_min'] < 0:
        raise ValueError('accel_min (up to %g) must be negative for every draw' % hi['u_min'])
    if not lo['u_max'] > 0:
        raise ValueError('accel_max (from %g) must be positive for every draw' % lo['u_max'])
    if not lo['v_star'] > 0:
        raise ValueError('speed_target (from %g) must be positive for every draw' % lo['v_star'])
    if not lo['h_star'] > 0:
        raise ValueError('headway_target (from %g) must be positive for every draw' % lo['h_star'])
    p = None
    if 'slowdown_prob' in config:
        p = config.getfloat('slowdown_prob')
        if not 0 <= p <= 1:
            raise ValueError('ENV_CONFIG.slowdown_prob = %g: needs 0 <= p <= 1' % p)
    return {'ranges': ranges, 'slowdown_prob': p}


class CACCEnv:
    def __init__(self, config, n_env=None, device=None, env0=0, n_env_total=None):
        """n_env overrides ENV_CONFIG.n_env.  A shard of a run over several processes holds the n_env envs
        env0 .. env0 + n_env - 1 of n_env_total: its random draws (initial conditions, per-env parameters) are keyed
        by the global env index, so they are those of the same envs in one process holding all n_env_total."""
        L.require_cuda()
        self._load_config(config)
        if n_env is not None:
            self.n_env = int(n_env)
        self.env0 = int(env0)
        self.n_env_total = self.n_env if n_env_total is None else int(n_env_total)
        if not (self.env0 >= 0 and self.env0 + self.n_env <= self.n_env_total):
            raise ValueError('envs %d .. %d are not inside the %d envs of the run'
                             % (self.env0, self.env0 + self.n_env - 1, self.n_env_total))
        if self.par_spec is not None and self.n_env_total == 1:
            raise ValueError('ENV_CONFIG keys %s (per-env scenario parameters) need batched training: set n_env > 1 '
                             '(VecTrainer); the one-env Trainer runs the nominal values only'
                             % ', '.join(env_par_keys(config)))
        self.device = torch.device(device if device is not None else 'cuda:%d' % torch.cuda.current_device())
        self.train_mode = True
        self.cur_episode = 0
        self.is_record = False
        self._init_space()
        self._alloc()
        if self.par_spec is not None:
            sp = self.par_spec
            logging.info('per-env scenario parameters, redrawn at every reset: %s; %s' % (
                ', '.join('%s in [%g, %g]' % (k, *sp['ranges'][f]) for k, f in PAR_KEYS.items()),
                'scenario %s' % self.name if sp['slowdown_prob'] is None else 'slowdown_prob %g' % sp['slowdown_prob']))
        # "required to achieve the same model initialization" (envs/cacc_env.py:21-22)
        np.random.seed(self.seed)

    # ---- configuration (envs/cacc_env.py:320-343) ---------------------------------------------
    def _load_config(self, config):
        self.dt = config.getfloat('control_interval_sec')
        self.T = int(config.getint('episode_length_sec') / self.dt)
        self.batch_size = config.getint('batch_size')
        self.h_min = config.getfloat('headway_min')
        self.h_star = config.getfloat('headway_target')
        self.h_norm = config.getfloat('norm_headway')
        self.h_s = config.getfloat('headway_st')
        self.h_g = config.getfloat('headway_go')
        self.v_max = config.getfloat('speed_max')
        self.v_star = config.getfloat('speed_target')
        self.v_norm = config.getfloat('norm_speed')
        self.u_min = config.getfloat('accel_min')
        self.u_max = config.getfloat('accel_max')
        self.name = config.get('scenario').split('_')[1]
        self.a = config.getfloat('reward_v')
        self.b = config.getfloat('reward_u')
        self.G = config.getfloat('collision_penalty')
        self.n_agent = config.getint('n_vehicle')
        self.agent = config.get('agent')
        self.coop_gamma = config.getfloat('coop_gamma')
        self.seed = config.getint('seed')
        self.init_test_seeds([int(s) for s in config.get('test_seeds').split(',')])
        self.n_env = config.getint('n_env', fallback=1)
        self.platoon_len = config.getint('platoon_len', fallback=self.n_agent)
        self.topology = config.get('topology', fallback='chain')
        if not (self.name.startswith('catchup') or self.name.startswith('slowdown')):
            raise ValueError('unknown CACC scenario %r' % self.name)
        self.par_spec = parse_env_par(config, self.h_min)

    def _init_space(self):
        if self.topology == 'grid':
            side = int(round(self.n_agent ** 0.5))
            assert side * side == self.n_agent, 'grid topology needs a square agent count'
            self.neighbor_mask, self.distance_mask = grid_masks(side)
        else:
            self.neighbor_mask, self.distance_mask = chain_masks(self.n_agent)
        self.n_a = 4
        self.n_a_ls = [4] * self.n_agent
        self.a_map = [(0, 0), (0.5, 0), (0, 0.5), (0.5, 0.5)]
        logging.info('action to h_go map:\n %r' % self.a_map)
        self.nbr = [np.where(self.neighbor_mask[i] == 1)[0] for i in range(self.n_agent)]
        self.n_s_ls = [5 * (1 if self.agent.startswith('ma2c') else 1 + len(self.nbr[i]))
                       for i in range(self.n_agent)]

    def _alloc(self):
        N, B, dev = self.n_agent, self.n_env, self.device
        P = N // self.platoon_len
        f64 = dict(dtype=torch.float64, device=dev)
        self.hs, self.vs, self.us = (torch.zeros(N, B, **f64) for _ in range(3))
        self.v_init = torch.zeros(P, B, **f64)
        self.t_dev = torch.zeros(B, dtype=torch.int32, device=dev)
        self.collision_dev = torch.zeros(B, dtype=torch.int32, device=dev)
        self.episode_dev = torch.zeros(B, dtype=torch.int32, device=dev)
        self.obs_stride = 8
        self.obs_dev = torch.zeros(N, B, self.obs_stride, dtype=torch.float32, device=dev)
        self.fp_dev = torch.full((N, B, self.n_a), 1.0 / self.n_a, dtype=torch.float32, device=dev)
        self.NR = 1 if self.coop_gamma < 0 else N
        self.reward_dev = torch.zeros(self.NR, B, **f64)
        self.greward_dev = torch.zeros(B, **f64)
        self.done_dev = torch.zeros(B, dtype=torch.float32, device=dev)
        self._action_dev = torch.zeros(N, B, dtype=torch.int32, device=dev)
        self._u01 = torch.zeros(P, B, **f64)
        self._mask0 = torch.zeros(B, dtype=torch.float32, device=dev)
        self._mask0[0] = 1.0
        c = L.CaccCfg()
        c.n_agent, c.platoon_len = N, self.platoon_len
        c.scenario = L.CATCHUP if self.name.startswith('catchup') else L.SLOWDOWN
        c.T, c.batch_size, c.global_reward = self.T, self.batch_size, int(self.coop_gamma < 0)
        c.dt, c.h_min, c.h_star, c.h_s, c.h_g = self.dt, self.h_min, self.h_star, self.h_s, self.h_g
        c.v_max, c.v_star, c.u_min, c.u_max = self.v_max, self.v_star, self.u_min, self.u_max
        c.rew_a, c.rew_b, c.G = self.a, self.b, self.G
        self.cfg = c
        # per-env scenario parameters: [B] rows of nmarl_cacc_env_par (8 x 8 bytes; the last holds the int32 scenario)
        self.env_par = None
        if self.par_spec is not None:
            self.env_par = torch.zeros(B, C.sizeof(L.CaccEnvPar) // 8, **f64)
            r = L.CaccParRanges()
            for k, f in enumerate(L.ENV_PAR_FIELDS):
                r.lo[k], r.hi[k] = self.par_spec['ranges'][f]
            p = self.par_spec['slowdown_prob']
            r.slowdown_prob = -1.0 if p is None else p
            self._par_ranges = r
        self.collision = False
        self.t = 0

    # ---- device-side API (no host copies) --------------------------------------------------------
    def reset_device(self, u01=None, mask=None, obs_out=None, fp_out=None, philox_seed=None):
        """Reset envs (all, or those with mask != 0).  u01: double [P,B] tensor or None (Philox keyed
        by (seed, env, episode counter))."""
        obs = self.obs_dev if obs_out is None else obs_out
        fp = self.fp_dev if fp_out is None else fp_out
        seed = int(self.cfg_seed if philox_seed is None else philox_seed) & (2 ** 64 - 1)
        if self.env_par is not None:
            # the reset envs draw their parameters for the episode they start (Philox keyed by seed, env, episode)
            L.check(L.lib().nmarl_cacc_draw_par_shard(C.byref(self.cfg), C.byref(self._par_ranges), self.n_env, seed,
                                                      L.ptr(self.episode_dev), L.ptr(mask), L.ptr(self.env_par),
                                                      L.stream(), self.env0), 'nmarl_cacc_draw_par_shard')
            L.check(L.lib().nmarl_cacc_reset_pe_shard(C.byref(self.cfg), L.ptr(self.env_par), self.n_env, L.ptr(u01),
                                                      L.ptr(mask), seed, L.ptr(self.episode_dev), L.ptr(self.hs),
                                                      L.ptr(self.vs), L.ptr(self.us), L.ptr(self.t_dev),
                                                      L.ptr(self.collision_dev), L.ptr(self.v_init), L.ptr(obs),
                                                      obs.shape[-1], L.ptr(fp), self.n_a, L.stream(), self.env0),
                    'nmarl_cacc_reset_pe_shard')
            return
        L.check(L.lib().nmarl_cacc_reset_shard(C.byref(self.cfg), self.n_env, L.ptr(u01), L.ptr(mask), seed,
                                               L.ptr(self.episode_dev), L.ptr(self.hs), L.ptr(self.vs), L.ptr(self.us),
                                               L.ptr(self.t_dev), L.ptr(self.collision_dev), L.ptr(self.v_init),
                                               L.ptr(obs), obs.shape[-1], L.ptr(fp), self.n_a, L.stream(), self.env0),
                'nmarl_cacc_reset_shard')

    def step_device(self, action, obs_out=None, reward_out=None, greward_out=None, done_out=None):
        """action int32 [N,B] device tensor.  Outputs default to the env's own buffers."""
        obs = self.obs_dev if obs_out is None else obs_out
        rew = self.reward_dev if reward_out is None else reward_out
        grew = self.greward_dev if greward_out is None else greward_out
        done = self.done_dev if done_out is None else done_out
        if self.env_par is not None:
            L.check(L.lib().nmarl_cacc_step_pe(C.byref(self.cfg), L.ptr(self.env_par), self.n_env, int(self.train_mode),
                                               L.ptr(action), L.ptr(self.hs), L.ptr(self.vs), L.ptr(self.us),
                                               L.ptr(self.t_dev), L.ptr(self.collision_dev), L.ptr(self.v_init),
                                               L.ptr(obs), obs.shape[-1], L.ptr(rew), L.ptr(grew), L.ptr(done),
                                               L.stream()), 'nmarl_cacc_step_pe')
            return
        L.check(L.lib().nmarl_cacc_step(C.byref(self.cfg), self.n_env, int(self.train_mode), L.ptr(action),
                                        L.ptr(self.hs), L.ptr(self.vs), L.ptr(self.us), L.ptr(self.t_dev),
                                        L.ptr(self.collision_dev), L.ptr(self.v_init), L.ptr(obs), obs.shape[-1],
                                        L.ptr(rew), L.ptr(grew), L.ptr(done), L.stream()), 'nmarl_cacc_step')

    # per-env device state kept in a snapshot, and the env axis of each ([agent][env] arrays: 1; [env] arrays: 0).
    # Not kept: _action_dev and _u01 (staging of the one-env host API, written before they are read) and _mask0
    # (a constant).
    SNAPSHOT_AXES = dict(hs=1, vs=1, us=1, v_init=1, t_dev=0, collision_dev=0, episode_dev=0, obs_dev=1, fp_dev=1,
                         reward_dev=1, greward_dev=0, done_dev=0, env_par=0)

    def snapshot(self):
        """Host copy of every per-env device tensor: vehicle state, leader profile (v_init), step and episode counters,
        collision / done latches, the per-env parameter table and the env's own observation / reward buffers.
        -> {'envs': {name: tensor}, 'env_axis': {name: env axis}}."""
        envs = {k: getattr(self, k).cpu() for k in self.SNAPSHOT_AXES if getattr(self, k) is not None}
        return dict(envs=envs, env_axis={k: self.SNAPSHOT_AXES[k] for k in envs})

    def restore(self, snap):
        """Copy a snapshot (global env order) into this env's tensors in place: the envs env0 .. env0 + n_env - 1."""
        if ('env_par' in snap['envs']) != (self.env_par is not None):
            raise ValueError('the snapshot %s per-env scenario parameters and this config %s' % (
                'has' if 'env_par' in snap['envs'] else 'has no', 'has' if self.env_par is not None else 'has none'))
        envs = D.take_envs(snap['envs'], snap['env_axis'], self.env0, self.n_env)
        for k, v in envs.items():
            dst = getattr(self, k)
            if tuple(v.shape) != tuple(dst.shape):
                raise ValueError('snapshot tensor %s has shape %s, this env needs %s' % (k, tuple(v.shape), tuple(dst.shape)))
            dst.copy_(v)

    @property
    def cfg_seed(self):
        return getattr(self, '_cfg_seed', 0)

    def par_table(self):
        """Host copy of the per-env parameter table: {field: float64 [B]} and 'scenario': int32 [B].  Host sync."""
        t = self.env_par.cpu()
        out = {f: t[:, k].numpy() for k, f in enumerate(L.ENV_PAR_FIELDS)}
        out['scenario'] = t.view(torch.int32)[:, 2 * len(L.ENV_PAR_FIELDS)].numpy()
        return out

    def par_stats(self, tab=None):
        """Mean, min and max over the batch of every drawn field (and of `slowdown`: 1 for a slow-down env), as one
        flat record {<field>_mean, <field>_min, <field>_max}.  tab: a table in the layout of par_table() (the rows of
        every shard of a sharded run); default this env's own.  Host sync."""
        tab = dict(self.par_table() if tab is None else tab)
        tab['slowdown'] = (tab.pop('scenario') == L.SLOWDOWN).astype(np.float64)
        rec = {}
        for f, v in tab.items():
            rec.update({f + '_mean': float(v.mean()), f + '_min': float(v.min()), f + '_max': float(v.max())})
        return rec

    # ---- reference API (host arrays, env 0 is "the" environment) -----------------------------------
    def _host_obs(self):
        base = self.obs_dev[:, 0, :5].double().cpu().numpy()
        if not self.agent.startswith('ia2c'):
            return [base[i] for i in range(self.n_agent)]
        # ia2c_fp: neighbour fingerprints are attached at the end of the state array (cacc_env.py:74-77)
        fps = (lambda i: [np.asarray(self.fp[j], dtype=np.float64) for j in self.nbr[i]]) if self.agent == 'ia2c_fp' else (lambda i: [])
        return [np.concatenate([base[i]] + [base[j] for j in self.nbr[i]] + fps(i)) for i in range(self.n_agent)]

    def reset(self, gui=False, test_ind=-1):
        """envs/cacc_env.py:166-189: seed selection, np.random.seed, ``seed += 1`` on every reset;
        one np.random.rand() drives the initial condition of env 0.  Envs b>0 (n_env > 1) draw
        their uniform from Philox keyed by (seed used, env, episode)."""
        self.cur_episode += 1
        if self.train_mode:
            seed = self.seed
        elif test_ind < 0:
            seed = self.seed - 1
        else:
            seed = self.test_seeds[test_ind]
        np.random.seed(seed)
        self.seed += 1
        # NB the reference tests the already-incremented attribute (cacc_env.py:290,311); the only
        # config seed reaching the deterministic branch (-1) is rejected by np.random.seed above.
        u = np.random.rand()
        if self.n_env > 1:
            self.reset_device(u01=None, philox_seed=seed)
            self.episode_dev[0] -= 1          # env 0 is reset again below; count its episode once
        # env 0: the reference's single np.random.rand(); further platoons (grid stub only) draw their own
        self._u01[:, 0] = torch.as_tensor([u] + [np.random.rand() for _ in range(self._u01.shape[0] - 1)],
                                          dtype=torch.float64)
        self.reset_device(u01=self._u01, mask=self._mask0)
        self.collision = False
        self.t = 0
        self.fp = np.ones((self.n_agent, self.n_a)) / self.n_a
        self.rewards = [0]
        if self.is_record:                       # the traffic log starts with the reset state (cacc_env.py:183-188)
            self._trace = [torch.stack([self.hs[:, 0], self.vs[:, 0], self.us[:, 0]]).cpu().numpy()]
        return self._host_obs()

    def step(self, action):
        """envs/cacc_env.py:191-242 for env 0 (all envs take the same action vector when n_env > 1)."""
        a = torch.as_tensor(np.asarray(action, dtype=np.int32)).to(self.device)
        self._action_dev.copy_(a[:, None].expand(-1, self.n_env))
        self.step_device(self._action_dev)
        out = torch.cat([self.reward_dev[:, 0], self.greward_dev[:1], self.done_dev[:1].double(),
                         self.collision_dev[:1].double()]).cpu().numpy()
        reward = out[0] if self.NR == 1 else out[:self.NR].copy()
        global_reward, done = out[self.NR], bool(out[self.NR + 1])
        self.collision = bool(out[self.NR + 2])
        self.t += 1
        self.rewards.append(global_reward)
        ob = self._host_obs()
        if self.is_record:
            self._log_control_data(action, global_reward)
            self._record_step()
            if done:
                self._log_traffic_data()
        return ob, reward, done, global_reward

    def get_fingerprint(self):
        return self.fp

    def update_fingerprint(self, fp):
        self.fp = fp

    def get_neighbor_action(self, action):
        action = np.asarray(action)
        return [action[self.neighbor_mask[i] == 1] for i in range(self.n_agent)]

    def terminate(self):
        return

    def collect_tripinfo(self):
        return

    def init_test_seeds(self, test_seeds):
        self.test_num = len(test_seeds)
        self.test_seeds = test_seeds

    # ---- evaluation records (envs/cacc_env.py:81-137) -------------------------------------------------
    def init_data(self, is_record, record_stats, output_path):
        self.is_record = is_record
        self.output_path = output_path
        if self.is_record:
            self.control_data = []
            self.traffic_data = []
            self._trace = []

    def _record_step(self):
        self._trace.append(torch.stack([self.hs[:, 0], self.vs[:, 0], self.us[:, 0]]).cpu().numpy())

    def _log_control_data(self, action, global_reward):
        self.control_data.append(control_record(self.cur_episode, self.t, self.dt, action, global_reward))

    def _log_traffic_data(self):
        self.traffic_data.append(traffic_frame(self.cur_episode, np.array(self._trace), self.rewards, self.dt))

    def output_data(self):
        if not self.is_record:
            logging.error('Env: no record to output!')
            return
        write_records(self.output_path, self.name, self.agent, self.control_data, self.traffic_data)


# ---- record formats (envs/cacc_env.py:81-112); shared by CACCEnv and the batched evaluator (utils.py) ---------------
def control_record(episode, t, dt, action, global_reward):
    """One row of <scenario>_<agent>_control.csv: step t (1-based) of episode `episode`."""
    return {'episode': episode, 'time_sec': t * dt, 'step': t, 'action': ','.join(['%d' % a for a in action]),
            'reward': global_reward}


def traffic_frame(episode, tr, rewards, dt):
    """The rows of <scenario>_<agent>_traffic.csv for one episode.  tr: float64 [steps + 1, 3, N] = (hs, vs, us) of
    the reset state and of every step; rewards: the steps + 1 global rewards, the reset's 0 first."""
    import pandas as pd
    hs, vs, us = tr[:, 0], tr[:, 1], tr[:, 2]
    df = pd.DataFrame()
    df['episode'] = np.ones(len(hs)) * episode
    df['time_sec'] = np.arange(len(hs)) * dt
    df['reward'] = np.array(rewards)
    df['lead_headway_m'] = hs[:, 0]
    df['avg_headway_m'] = np.mean(hs[:, 1:], axis=1)
    df['std_headway_m'] = np.std(hs[:, 1:], axis=1)
    df['avg_speed_mps'] = np.mean(vs, axis=1)
    df['std_speed_mps'] = np.std(vs, axis=1)
    df['avg_accel_mps2'] = np.mean(us, axis=1)
    df['std_accel_mps2'] = np.std(us, axis=1)
    for i in range(tr.shape[2]):
        df['headway_%d_m' % (i + 1)] = hs[:, i]
        df['velocity_%d_mps' % (i + 1)] = vs[:, i]
        df['accel_%d_mps2' % (i + 1)] = us[:, i]
    return df


def write_records(output_path, name, agent, control_data, traffic_data):
    """control_data: list of control_record rows; traffic_data: list of traffic_frame frames, in episode order."""
    import pandas as pd
    pd.DataFrame(control_data).to_csv(output_path + ('%s_%s_control.csv' % (name, agent)))
    pd.concat(traffic_data).to_csv(output_path + ('%s_%s_traffic.csv' % (name, agent)))
