"""IA2C / MA2C agent API -- drop-in mirror of the reference's agents/models.py.

Same constructor ``(n_s_ls, n_a_ls, neighbor_mask, distance_mask, coop_gamma, total_step,
model_config, seed=0)`` and methods ``forward / add_transition / backward / reset / save /
load`` (agents/models.py:15-158,191-258,278-309), with host lists / NumPy arrays in and NumPy
out, so ``Trainer`` and ``main.py`` run unchanged.  Underneath, everything is executed by the
libnmarl CUDA kernels through :class:`PolicyEngine`; there is no TF session (``sess`` is None).

Extra keyword arguments (not in the reference): ``n_env`` parallel environments (default 1,
which is exactly the reference), ``device``, ``obs_mode`` (IA2C only, see ModelLayout), and for one shard of a
run over several processes ``env0`` / ``n_env_total`` (the global index of this shard's first env, the run's env
count: the sampled actions are keyed by the global env index).
With ``n_env > 1`` use the batched entry points ``rollout`` / ``update`` (device resident).
"""
import logging
import os

import numpy as np
import torch

from .. import _lib as L
from ..layout import HeteroLayout, ModelLayout
from ..resume import atomic_save
from .engine import PolicyEngine
from .utils import Scheduler


class IA2C:
    """Independent A2C: per-agent LSTM policy, loss, clip and optimizer (agents/models.py:15-158)."""
    variant = 'ia2c'

    def __init__(self, n_s_ls, n_a_ls, neighbor_mask, distance_mask, coop_gamma,
                 total_step, model_config, seed=0, n_env=1, device=None, obs_mode=None, flat_params=None, env0=0,
                 n_env_total=None):
        self.name = self.variant
        self._init_algo(n_s_ls, n_a_ls, neighbor_mask, distance_mask, coop_gamma, total_step, seed,
                        model_config, n_env, device, obs_mode, flat_params, env0, n_env_total)

    # ---- construction (agents/models.py:84-158, 246-258) ------------------------------------------
    def _init_algo(self, n_s_ls, n_a_ls, neighbor_mask, distance_mask, coop_gamma, total_step, seed,
                   model_config, n_env, device, obs_mode, flat_params, env0=0, n_env_total=None):
        self.n_s_ls, self.n_a_ls = list(n_s_ls), list(n_a_ls)
        # agents/models.py:89-97: agents are "identical" iff all action spaces are equal; otherwise inputs are
        # zero-padded to the widest agent and the *_hetero layers slice each agent's valid part
        self.identical_agent = max(self.n_a_ls) == min(self.n_a_ls)
        if self.identical_agent:
            self.n_s, self.n_a = self.n_s_ls[0], self.n_a_ls[0]
        else:
            self.n_s, self.n_a = max(self.n_s_ls), max(self.n_a_ls)
        self.neighbor_mask = np.asarray(neighbor_mask)
        self.n_agent = len(self.neighbor_mask)
        self.reward_clip = model_config.getfloat('reward_clip')
        self.reward_norm = model_config.getfloat('reward_norm')
        self.n_step = model_config.getint('batch_size')
        self.n_fc = model_config.getint('num_fc')
        self.n_lstm = model_config.getint('num_lstm')
        self.n_env = int(n_env)
        self.sess = None
        if not self.identical_agent and self.variant in ('ia2c', 'ia2c_fp') and obs_mode not in (None, 'concat'):
            raise ValueError('heterogeneous %s agents read their own observation rows as given (obs_mode concat)'
                             % self.variant)
        if obs_mode is None:
            obs_mode = 'concat' if self.variant == 'ia2c' else 'gather'
        own_n_s_ls = list(self.n_s_ls)
        if self.variant == 'ia2c_fp':     # "neighborhood policies are included in local state" (agents/models.py:172-188)
            self.n_s_ls = [n + sum(self.n_a_ls[j] for j in np.where(self.neighbor_mask[i] == 1)[0])
                           for i, n in enumerate(self.n_s_ls)]
        if self.identical_agent:
            self.layout = ModelLayout(self.variant, self.n_s_ls, self.n_a, self.neighbor_mask,
                                      n_h=self.n_lstm, n_fc=self.n_fc, obs_mode=obs_mode)
        else:
            # IA2C / IA2C_FP read each agent's own observation row as given (IA2C_FP: the part in front of the
            # fingerprints); the MA2C family and IA2C_CU pad it to max(n_s_ls)
            self.layout = HeteroLayout(self.variant, own_n_s_ls, self.n_a_ls, self.neighbor_mask,
                                       n_h=self.n_lstm, n_fc=self.n_fc)
        self.nbr = self.layout.nbr
        hp = dict(v_coef=0.5, e_coef=0.01, max_grad_norm=40.0, alpha=0.99, epsilon=1e-5, gamma=0.99,
                  reward_norm=self.reward_norm, reward_clip=self.reward_clip)
        self.total_step = total_step
        if total_step:
            lr_init = model_config.getfloat('lr_init')
            lr_decay = model_config.get('lr_decay')
            if lr_decay == 'constant':
                self.lr_scheduler = Scheduler(lr_init, decay=lr_decay)
            else:
                self.lr_scheduler = Scheduler(lr_init, model_config.getfloat('lr_min'), self.total_step, decay=lr_decay)
            hp.update(v_coef=model_config.getfloat('value_coef'), e_coef=model_config.getfloat('entropy_coef'),
                      max_grad_norm=model_config.getfloat('max_grad_norm'), alpha=model_config.getfloat('rmsp_alpha'),
                      epsilon=model_config.getfloat('rmsp_epsilon'), gamma=model_config.getfloat('gamma'))
        # weights come from the global NumPy stream in the reference's variable-creation order
        self.engine = PolicyEngine(self.layout, self.n_env, self.n_step, hp, flat_params=flat_params, device=device,
                                   rng_seed=seed, distance_mask=distance_mask, coop_gamma=coop_gamma, env0=env0,
                                   n_env_total=n_env_total)
        self.device = self.engine.device
        self._reset_host_buffer(False)
        e = self.engine
        self._one = dict(obs=e.obs_buf[0], fp=e.fp_buf[0], done=e.done_buf[0], act=e.act_buf[0], v=e.val_buf[0])

    # ---- host staging of one transition batch (the reference's OnPolicyBuffer) -----------------------
    def _reset_host_buffer(self, done):
        self._obs, self._ps, self._acts, self._rs, self._vs, self._dones = [], [], [], [], [], [done]

    def _pack_obs(self, obs):
        """list of N per-agent arrays -> float32 [N, obs_stride] rows (own features, or the caller's
        pre-concatenated vector in IA2C 'concat' mode)."""
        S = self.layout.obs_stride
        out = np.zeros((self.n_agent, S), dtype=np.float32)
        for i in range(self.n_agent):
            o = np.asarray(obs[i], dtype=np.float32).ravel()
            if self.layout.obs_mode == 'gather':
                w = min(len(o), self.layout.base_n_s)
            elif self.variant == 'ia2c_fp':     # heterogeneous IA2C_FP: the fingerprints behind it go to _ps_from_obs
                w = self.layout.n_s_ls[i]
            else:
                w = len(o)
            out[i, :w] = o[:w]              # shorter rows (heterogeneous agents) stay zero-padded (agents/models.py:229-235)
        return out

    def _upload_step(self, obs, done, ps):
        assert self.n_env == 1, 'the list-based API drives one environment; use rollout()/update() for n_env > 1'
        s = self._one
        s['obs'].copy_(torch.from_numpy(self._pack_obs(obs))[:, None, :])
        s['done'].fill_(float(bool(done)))
        if ps is not None:
            s['fp'].copy_(torch.as_tensor(self._pad_ps(ps))[:, None, :])

    # ---- reference API ---------------------------------------------------------------------------------
    def forward(self, obs, done, nactions=None, out_type='p'):
        """agents/models.py:44-51 -> list of N arrays (pi_i) or N scalars (v_i)."""
        e, s = self.engine, self._one
        ps = self._ps_from_obs(obs)
        self._upload_step(obs, done, ps)
        fp = None if ps is None else s['fp']
        if out_type.startswith('p'):
            e.step_p(s['obs'], fp, s['done'], e.pi_tmp)
            pi = e.pi_tmp[:, 0].cpu().numpy()
            return [pi[i, :self.n_a_ls[i]] for i in range(self.n_agent)]      # heterogeneous agents: tight widths
        a = np.zeros(self.n_agent, dtype=np.int32)
        for i in range(self.n_agent):
            for k, j in enumerate(self.nbr[i]):
                a[j] = int(nactions[i][k])
        s['act'].copy_(torch.from_numpy(a)[:, None])
        e.step_v(s['obs'], fp, s['done'], s['act'], s['v'])
        v = s['v'][:, 0].cpu().numpy()
        return [v[i] for i in range(self.n_agent)]

    def _ps_from_obs(self, obs):
        """Fingerprints carried inside the observation (only IA2C_FP has them)."""
        return None

    def _pad_ps(self, ps):
        """[N, n_a] float32; heterogeneous agents hand over a list of per-agent policies of different lengths,
        zero-padded to the widest action space (agents/models.py:229-235)."""
        if self.identical_agent:
            return np.asarray(ps, dtype=np.float32)
        out = np.zeros((self.n_agent, self.n_a), dtype=np.float32)
        for i, q in enumerate(ps):
            q = np.asarray(q, dtype=np.float32).ravel()
            out[i, :len(q)] = q
        return out

    def add_transition(self, ob, naction, action, reward, value, done):
        """agents/models.py:26-32 (reward norm/clip happen inside the returns kernel)."""
        self._obs.append(self._pack_obs(ob)); self._ps.append(self._ps_from_obs(ob)); self._acts.append(np.asarray(action, dtype=np.int32))
        self._rs.append(reward); self._vs.append(np.asarray(value, dtype=np.float32)); self._dones.append(bool(done))

    def backward(self, Rends, dt=0, summary_writer=None, global_step=None):
        """agents/models.py:34-42 / 211-215: lr schedule -> returns -> training pass -> optimizer."""
        cur_lr = self.lr_scheduler.get(self.n_step)
        e = self.engine
        T = len(self._rs)
        e.T_cur = T
        e.obs_buf[:T].copy_(torch.from_numpy(np.stack(self._obs))[:, :, None, :])
        if self._ps[0] is not None:
            e.fp_buf[:T].copy_(torch.from_numpy(np.stack(self._ps))[:, :, None, :])
        e.act_buf[:T].copy_(torch.from_numpy(np.stack(self._acts))[:, :, None])
        e.val_buf[:T].copy_(torch.from_numpy(np.stack(self._vs))[:, :, None])
        r = np.stack([np.broadcast_to(np.asarray(x, dtype=np.float64), (e.NR,)) for x in self._rs])
        e.rew_buf[:T].copy_(torch.from_numpy(r)[:, :, None])
        e.done_buf[:T + 1].copy_(torch.tensor(self._dones, dtype=torch.float32)[:, None])
        e.R_end.copy_(torch.as_tensor(np.asarray(Rends, dtype=np.float32))[:, None])
        e.update(cur_lr)
        self._reset_host_buffer(self._dones[-1])
        if summary_writer is not None:
            self._write_summary(summary_writer, cur_lr, global_step)

    def _write_summary(self, writer, lr, global_step):
        """Scalar tags of agents/policies.py:41-47 / 266-273."""
        ls = self.engine.losses()
        norms = self.engine.norm_out.cpu().numpy()
        per_agent = bool(self.engine.model.per_agent_norm)
        names = ['lstm_%d' % i for i in range(self.n_agent)] if per_agent else [self.layout_scope()]
        for k, name in enumerate(names[:1] if per_agent else names):
            sel = slice(k, k + 1) if per_agent else slice(None)
            pl, vl, el = ls['policy_loss'][sel].sum(), ls['value_loss'][sel].sum(), ls['entropy_loss'][sel].sum()
            writer.add_scalar('loss/%s_entropy_loss' % name, el, global_step)
            writer.add_scalar('loss/%s_policy_loss' % name, pl, global_step)
            writer.add_scalar('loss/%s_value_loss' % name, vl, global_step)
            writer.add_scalar('loss/%s_total_loss' % name, pl + vl + el, global_step)
            writer.add_scalar('train/%s_lr' % name, lr, global_step)
            writer.add_scalar('train/%s_gradnorm' % name, float(norms[k]), global_step)

    def layout_scope(self):
        return {'ma2c_nc': 'nc', 'ma2c_ic3': 'ic3', 'ma2c_dial': 'dial', 'ma2c_cu': 'cu'}.get(self.variant, 'lstm')

    def reset(self):
        self.engine.reset_states()

    # ---- checkpoints (agents/models.py:53-82; own on-disk format, same naming rule) ---------------------
    def save(self, model_dir, global_step):
        """<model_dir>/checkpoint-<step>.pt, written under a temporary name and renamed (resume.atomic_save)."""
        e = self.engine
        atomic_save({'variant': self.variant, 'names': [n for n, _, _ in self.layout.entries],
                     'params': e.params.cpu(), 'ms': e.ms.cpu(), 'global_step': int(global_step)},
                    model_dir + 'checkpoint-%d.pt' % int(global_step))

    def load(self, model_dir, checkpoint=None):
        save_file, save_step = None, 0
        if os.path.exists(model_dir):
            if checkpoint is None:
                for file in os.listdir(model_dir):
                    if file.startswith('checkpoint'):
                        prefix = file.split('.')[0]
                        tokens = prefix.split('-')
                        if len(tokens) != 2:
                            continue
                        cur_step = int(tokens[1])
                        if cur_step > save_step:
                            save_file, save_step = prefix, cur_step
            else:
                save_file = 'checkpoint-' + str(int(checkpoint))
        if save_file is not None and os.path.exists(model_dir + save_file + '.pt'):
            ck = torch.load(model_dir + save_file + '.pt', map_location='cpu')
            self.engine.params.copy_(ck['params']); self.engine.ms.copy_(ck['ms'])
            self.engine.repack(); self.engine._refresh_msg()
            logging.info('Checkpoint loaded: %s' % save_file)
            return True
        logging.error('Can not find old checkpoint for %s' % model_dir)
        return False

    # ---- weights by reference variable name (tests, importers) ------------------------------------------
    def get_weights(self):
        return self.layout.unpack(self.engine.params.cpu().numpy())

    def set_weights(self, params):
        self.engine.params.copy_(torch.from_numpy(self.layout.pack(params)))
        self.engine.repack()
        self.engine._refresh_msg()

    # ---- batched entry points (n_env >= 1, device resident) ----------------------------------------------
    def rollout(self, env, **kw):
        self.engine.rollout(env, **kw)

    def update(self):
        # the schedule counts environment steps: n_step steps of every env on every rank per update
        self.engine.update(self.lr_scheduler.get(self.n_step * self.n_env * self.engine.world))


class IA2C_FP(IA2C):
    """Fingerprint IA2C (agents/models.py:161-188): FPPolicy encodes the neighbours' last policies, which the
    environment appends to each observation (envs/cacc_env.py:74-77), with a second fc layer.  The kernels
    gather observations and fingerprints per neighbour on the device, so the host splits the reference's
    concatenated observation back into own features and one policy row per agent.  With heterogeneous agents each
    neighbour's fingerprint is n_a_ls[j] wide, and the own features are the first n_s_ls[i] entries as given."""
    variant = 'ia2c_fp'

    def _ps_from_obs(self, obs):
        if not self.identical_agent:
            # agent i's observation = its own n_s_ls[i] features, then neighbour j's policy (n_a_ls[j] wide) for every
            # neighbour in ascending order (agents/models.py:181-184).  Rows are zero-padded to max(n_a_ls): a padded
            # fingerprint entry must be exactly 0, as it meets fcp rows that are padding.
            ps = np.zeros((self.n_agent, self.n_a), dtype=np.float32)
            for i in range(self.n_agent):
                o = np.asarray(obs[i], dtype=np.float32).ravel()
                off = self.layout.n_s_ls[i]
                for j in self.nbr[i]:
                    ps[j, :self.n_a_ls[j]] = o[off: off + self.n_a_ls[j]]
                    off += self.n_a_ls[j]
            return ps
        ps = np.full((self.n_agent, self.n_a), 1.0 / self.n_a, dtype=np.float32)
        b = self.layout.base_n_s
        for i in range(self.n_agent):
            o = np.asarray(obs[i], dtype=np.float32).ravel()
            n_x = b * (1 + len(self.nbr[i]))
            for k, j in enumerate(self.nbr[i]):
                ps[j] = o[n_x + k * self.n_a: n_x + (k + 1) * self.n_a]
        return ps


class MA2C_NC(IA2C):
    """NeurComm (agents/models.py:191-258): centralised graph over all agents."""
    variant = 'ma2c_nc'

    def forward(self, obs, done, ps, actions=None, out_type='p'):
        """agents/models.py:217-224 -> pi [N, n_a] or v [N]."""
        e, s = self.engine, self._one
        self._upload_step(obs, done, ps)
        if out_type.startswith('p'):
            e.step_p(s['obs'], s['fp'], s['done'], e.pi_tmp)
            pi = e.pi_tmp[:, 0].cpu().numpy()
            if self.identical_agent:
                return pi
            return [pi[i, :self.n_a_ls[i]] for i in range(self.n_agent)]     # pi_ls of agents/policies.py:296
        s['act'].copy_(torch.as_tensor(np.asarray(actions, dtype=np.int32))[:, None])
        e.step_v(s['obs'], s['fp'], s['done'], s['act'], s['v'])
        return s['v'][:, 0].cpu().numpy()

    def add_transition(self, ob, p, action, reward, value, done):
        """agents/models.py:198-209"""
        self._obs.append(self._pack_obs(ob)); self._ps.append(self._pad_ps(p))
        self._acts.append(np.asarray(action, dtype=np.int32)); self._rs.append(reward)
        self._vs.append(np.asarray(value, dtype=np.float32)); self._dones.append(bool(done))


class MA2C_IC3(MA2C_NC):
    """CommNet (agents/models.py:278-292); config key ``ma2c_ic3``."""
    variant = 'ma2c_ic3'


class MA2C_DIAL(MA2C_NC):
    """DIAL (agents/models.py:295-309)."""
    variant = 'ma2c_dial'


class IA2C_CU(MA2C_NC):
    """Consensus update (agents/models.py:261-275, config key ``ma2c_cu``): per-agent fc + LSTM on the agent's
    own observation inside one graph (one loss, one global clip); after every optimizer step each agent's
    LSTM weights are replaced by the mean over itself and its neighbours (nmarl_consensus_update)."""
    variant = 'ma2c_cu'
