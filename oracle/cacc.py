"""CPU oracle: CACC platoon environment (float64 NumPy restatement).

TEST INFRASTRUCTURE -- see ``oracle/__init__.py``.  PINNED against the unmodified
reference env through ``tests/golden/env_*.npz``.

Follows ``/root/reference/envs/cacc_env.py``:
  * optimal-velocity curve + OVM acceleration   -- cacc_env.py:360-385
  * speed constraint / trapezoid headway update -- cacc_env.py:24-38, 191-223
  * reward + collision latch                    -- cacc_env.py:40-52
  * per-vehicle 5-feature observation           -- cacc_env.py:54-79
  * done rule / global reward / coop_gamma<0    -- cacc_env.py:225-242
  * reset, seed stepping, catch-up / slow-down  -- cacc_env.py:166-189, 285-318
  * chain adjacency / distance / n_s            -- cacc_env.py:253-283

The arithmetic is kept scalar and in the reference's operation order so the
float64 results are bit-identical (checked by tests/test_oracle_env.py).
"""

import numpy as np

COLLISION_WT = 5          # cacc_env.py:9
COLLISION_HEADWAY = 10    # cacc_env.py:10
VDIFF = 5                 # cacc_env.py:11
A_MAP = ((0.0, 0.0), (0.5, 0.0), (0.0, 0.5), (0.5, 0.5))   # cacc_env.py:275


def chain_masks(n):
    """Chain adjacency and |i-j| distance (cacc_env.py:254-267)."""
    nb = np.zeros((n, n), dtype=int)
    for i in range(n):
        if i > 0:
            nb[i, i - 1] = 1
        if i < n - 1:
            nb[i, i + 1] = 1
    idx = np.arange(n)
    dist = np.abs(idx[:, None] - idx[None, :]).astype(int)
    return nb, dist


class CACCParams:
    """ENV_CONFIG keys (cacc_env.py:320-343).  ``cfg`` is a mapping of strings."""

    def __init__(self, cfg):
        g = lambda k: float(cfg[k])
        self.dt = g('control_interval_sec')
        self.T = int(int(cfg['episode_length_sec']) / self.dt)
        self.batch_size = int(cfg['batch_size'])
        self.h_min = g('headway_min')
        self.h_star = g('headway_target')
        self.h_s = g('headway_st')
        self.h_g = g('headway_go')
        self.v_max = g('speed_max')
        self.v_star = g('speed_target')
        self.u_min = g('accel_min')
        self.u_max = g('accel_max')
        self.name = cfg['scenario'].split('_')[1]
        self.a = g('reward_v')
        self.b = g('reward_u')
        self.G = g('collision_penalty')
        self.n_agent = int(cfg['n_vehicle'])
        self.agent = cfg['agent']
        self.coop_gamma = g('coop_gamma')
        self.seed = int(cfg['seed'])
        self.test_seeds = [int(s) for s in str(cfg['test_seeds']).split(',')]


class OracleCACC:
    """Same public surface as the reference ``CACCEnv`` (SURVEY 8b, env row)."""

    def __init__(self, cfg):
        p = CACCParams(cfg)
        self.p = p
        for k, v in vars(p).items():
            setattr(self, k, v)
        self.test_num = len(self.test_seeds)
        self.train_mode = True
        self.cur_episode = 0
        self.n_a = 4
        self.n_a_ls = [4] * self.n_agent
        self.neighbor_mask, self.distance_mask = chain_masks(self.n_agent)
        per = lambda i: 1 if self.agent.startswith('ma2c') else 1 + int(self.neighbor_mask[i].sum())
        self.n_s_ls = [5 * per(i) for i in range(self.n_agent)]
        np.random.seed(self.seed)            # cacc_env.py:21-22

    # ---- dynamics -----------------------------------------------------------------
    def _vh(self, h):
        """cacc_env.py:360-369"""
        if h <= self.h_s:
            return 0
        if h < self.h_g:
            return self.v_max / 2 * (1 - np.cos(np.pi * (h - self.h_s) / (self.h_g - self.h_s)))
        return self.v_max

    def _lead(self, i, vs, t):
        return vs[i - 1] if i else self.v0s[t]

    def step(self, action):
        n = self.n_agent
        if self.collision:                    # cacc_env.py:193-194
            reward = -self.G * np.ones(n)
        else:
            v_new = np.empty(n)
            u_new = np.empty(n)
            for i in range(n):
                al, be = A_MAP[int(action[i])]
                v = self.vs_cur[i]
                u = al * (self._vh(self.hs_cur[i]) - v) + be * (self._lead(i, self.vs_cur, self.t) - v)
                vn = v + np.clip(u, self.u_min, self.u_max) * self.dt
                vn = np.clip(vn, 0, self.v_max)
                v_new[i] = vn
                u_new[i] = (vn - v) / self.dt
            h_new = np.empty(n)
            for i in range(n):
                if i == 0:
                    vl, vln = self.v0s[self.t], self.v0s[self.t + 1]
                else:
                    vl, vln = self.vs_cur[i - 1], v_new[i - 1]
                h_new[i] = self.hs_cur[i] + 0.5 * self.dt * (vl + vln - self.vs_cur[i] - v_new[i])
            self.hs_cur, self.vs_cur, self.us_cur = h_new, v_new, u_new
            reward = self._reward()
        self.t += 1
        global_reward = np.sum(reward)
        done = bool((self.collision and self.t % self.batch_size == 0) or self.t == self.T)
        if self.coop_gamma < 0:
            reward = global_reward
        return self._state(), reward, done, global_reward

    def _reward(self):
        if np.min(self.hs_cur) < self.h_min:            # cacc_env.py:42-44
            self.collision = True
            return -self.G * np.ones(self.n_agent)
        r = -(self.hs_cur - self.h_star) ** 2
        r = r + (-self.a * (self.vs_cur - self.v_star) ** 2)
        r = r + (-self.b * (self.us_cur) ** 2)
        if self.train_mode:
            r = r + (-COLLISION_WT * (np.minimum(self.hs_cur - COLLISION_HEADWAY, 0)) ** 2)
        else:
            r = r + 0
        return r

    def _veh_obs(self, i):
        """cacc_env.py:54-65 (uses the already-incremented t)."""
        v = self.vs_cur[i]
        vl = self._lead(i, self.vs_cur, self.t)
        return np.array([
            (v - self.v_star) / self.v_star,
            np.clip((vl - v) / VDIFF, -2, 2),
            np.clip((self._vh(self.hs_cur[i]) - v) / VDIFF, -2, 2),
            (self.hs_cur[i] + (vl - v) * self.dt - self.h_star) / self.h_star,
            self.us_cur[i] / self.u_max])

    def _state(self):
        base = [self._veh_obs(i) for i in range(self.n_agent)]
        if not self.agent.startswith('ia2c'):
            return base
        out = []
        for i in range(self.n_agent):
            nb = np.where(self.neighbor_mask[i] == 1)[0]
            parts = [base[i]] + [base[j] for j in nb]
            if self.agent == 'ia2c_fp':          # fingerprints go at the end (envs/cacc_env.py:74-77)
                parts += [self.fp[j] for j in nb]
            out.append(np.concatenate(parts))
        return out

    # ---- episode control ----------------------------------------------------------
    def reset(self, gui=False, test_ind=-1, u01=None):
        """u01 (tests only): use this uniform instead of the np.random.rand() draw."""
        self.cur_episode += 1
        if self.train_mode:
            seed = self.seed
        elif test_ind < 0:
            seed = self.seed - 1
        else:
            seed = self.test_seeds[test_ind]
        np.random.seed(seed)
        self.seed += 1
        self.t = 0
        n = self.n_agent
        h0 = np.ones(n) * self.h_star
        if self.name.startswith('catchup'):
            # NB: tests the already-incremented seed attribute (cacc_env.py:176 vs :290)
            h0[0] = self.h_star * 2 if not self.seed else self.h_star * (1.5 + (np.random.rand() if u01 is None else u01))
            v0 = np.ones(n) * self.v_star
            self.v0s = np.ones(self.T + 1) * self.v_star
        else:
            if not self.seed:
                v0 = np.ones(n) * 2 * self.v_star
            else:
                v0 = np.ones(n) * self.v_star * (1.5 + (np.random.rand() if u01 is None else u01))
            self.v0s = np.ones(self.T + 1) * self.v_star
            dec = np.linspace(v0[0], self.v_star, 300)
            # episodes shorter than the 300-step ramp keep its first T + 1 entries (the reference needs T >= 299)
            self.v0s[:len(dec)] = dec[:self.T + 1]
        self.collision = False
        self.hs_cur, self.vs_cur, self.us_cur = h0, v0, np.zeros(n)
        self.fp = np.ones((n, self.n_a)) / self.n_a
        return self._state()

    def get_fingerprint(self):
        return self.fp

    def update_fingerprint(self, fp):
        self.fp = fp

    def get_neighbor_action(self, action):
        action = np.asarray(action)
        return [action[self.neighbor_mask[i] == 1] for i in range(self.n_agent)]

    def terminate(self):
        return

    def init_test_seeds(self, test_seeds):
        self.test_num = len(test_seeds)
        self.test_seeds = test_seeds


def leader_speed(scenario, v_init, v_star, t):
    """Closed form of ``v0s[t]`` (cacc_env.py:299, 316-318) used by the CUDA kernel:
    catch-up: v*;  slow-down: np.linspace(v_init, v*, 300)[t] for t<300, then v*.
    np.linspace(a, b, 300)[t] == t * ((b - a) / 299) + a for t < 299, and b at t == 299.
    """
    if scenario.startswith('catchup') or t >= 300:
        return v_star
    if t == 299:
        return v_star
    step = (v_star - v_init) / 299.0
    return t * step + v_init


def np_pairwise_sum(x):
    """np.sum order for a contiguous float64 vector of length < 128
    (numpy pairwise_sum: sequential for n < 8, 8 strided accumulators otherwise)."""
    n = len(x)
    if n < 8:
        res = 0.0
        for v in x:
            res += v
        return res
    r = [x[j] for j in range(8)]
    i = 8
    while i < n - (n % 8):
        for j in range(8):
            r[j] += x[i + j]
        i += 8
    res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    while i < n:
        res += x[i]
        i += 1
    return res
