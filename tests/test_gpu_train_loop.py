"""GPU: the batched training loop (`VecTrainer`) against the oracle, update by update, across episode boundaries.

Every kernel call is pinned elsewhere; this file pins what happens BETWEEN them over several updates: the optimizer
step and the refresh of the tensor-core operand copies (`repack`) and of DIAL's cached messages, RMSProp slots carried
from update to update, the learning-rate schedule, the Philox counter (T + 1 p-calls per update), and the hand-over
of `_one_update` -- slot T becomes slot 0, the envs whose episode ended restart (LSTM state, env state, fingerprints)
while the others keep going, and states_bw := states_fw.

Each case drives the real `VecTrainer`, `CACCEnv` and agent class eagerly for K updates.  Episodes are 3 updates
long, and after the first update every third env is restarted with the hand-over's own calls, so the time limit ends
one group's episodes at update 3 and the other's at update 4 (collisions cannot be relied on for that: random
policies on these platoons do not collide within a few hundred steps).  Every update is judged from the kernel's own
state at its start (teacher forcing), so errors never compound and the fp32 trajectories never drift apart:
  1. rollout   fp32 oracle (oracle/nets.py) over t = 0..T incl. the bootstrap: pi, v, R_end; actions against the
               Philox stream (tests/philox_ref.py) on the kernel's pi, and the oracle's draw away from cdf steps
  2. env       one persistent NumPy env (oracle/cacc.py) per env, driven by the kernel's actions
  3. returns   float64 `nstep_returns` on the kernel's rewards and values
  4. gradient  float64 autograd from the pre-update weights and states_bw; losses
  5. apply     float64 clip + TF-RMSProp (+ consensus update) from the kernel's pre-update weights and slots
  6. hand-over checked at the start of the next update (and right after `apply`)
"""
import numpy as np
import pytest
import torch

import philox_ref as P
from gpu_common import oracle_obs
from helpers import load_cfg, random_params
from oracle import nets
from oracle.buffers import Scheduler, nstep_returns
from oracle.cacc import OracleCACC
from test_gpu_tc_paths import RoundoffScale

pytestmark = pytest.mark.gpu

T, K = 10, 6                    # steps per update, updates per case
EPISODE_SEC = 3                 # 30 steps at dt = 0.1: an episode is 3 updates
LR_INIT, LR_MIN, HORIZON = 1e-2, 1e-3, 20      # linear decay over HORIZON updates: the lr changes every update
CLIP_ON, CLIP_OFF = 0.5, 1e3    # global norms of these models at scale-0.3 weights are ~1-6 per group
MODEL_SEED = 5                  # Philox key of the action stream (the env resets use the config seed, 12)
MSG_TOL = 1e-6                  # DIAL's cached messages against float64 from the kernel's own h and weights
CFGS = [('ma2c_nc', 'config_ma2c_nc_catchup.ini'), ('ma2c_ic3', 'config_ma2c_cnet_slowdown.ini'),
        ('ma2c_dial', 'config_ma2c_dial_catchup.ini'), ('ia2c_fp', 'config_ia2c_fp_slowdown.ini'),
        ('ia2c', 'config_ia2c_slowdown.ini'), ('ma2c_cu', 'config_ia2c_cu_catchup.ini')]
CASES = []
for _k, (_agent, _ini) in enumerate(CFGS):
    for _B in (128, 37):        # tensor cores (fused saved rollout); FP32-FFMA with a ragged 64-row tile
        _clip = (_k + (_B == 37)) % 2 == 0          # every config runs once with the clip active and once without
        CASES.append(pytest.param(_agent, _ini, _B, True, _clip,
                                  id='%s-B%d-%s' % (_agent, _B, 'clip' if _clip else 'noclip')))
# the unfused tensor-core path: backward runs the training forward from states_bw (the fused one never reads it)
CASES.append(pytest.param('ma2c_nc', 'config_ma2c_nc_catchup.ini', 128, False, False, id='ma2c_nc-B128-unfused'))


def _make(agent, ini, B, clip, graph=False):
    from deeprl_network_b200.agents.models import IA2C, IA2C_CU, IA2C_FP, MA2C_DIAL, MA2C_IC3, MA2C_NC
    from deeprl_network_b200.envs.cacc_env import CACCEnv
    from deeprl_network_b200.utils import VecTrainer
    cls = {'ma2c_nc': MA2C_NC, 'ia2c': IA2C, 'ma2c_ic3': MA2C_IC3, 'ma2c_dial': MA2C_DIAL, 'ia2c_fp': IA2C_FP,
           'ma2c_cu': IA2C_CU}[agent]
    cp = load_cfg(ini, n_env=B, batch_size=T, episode_length_sec=EPISODE_SEC)
    mc = cp['MODEL_CONFIG']
    mc['batch_size'], mc['lr_init'], mc['lr_min'], mc['lr_decay'] = str(T), str(LR_INIT), str(LR_MIN), 'linear'
    mc['max_grad_norm'] = str(CLIP_ON if clip else CLIP_OFF)
    env = CACCEnv(cp['ENV_CONFIG'])
    kw = dict(obs_mode='gather') if agent == 'ia2c' else {}
    total_step = HORIZON * T * B
    model = cls(env.n_s_ls, env.n_a_ls, env.neighbor_mask, env.distance_mask, env.coop_gamma, total_step, mc,
                seed=MODEL_SEED, n_env=B, **kw)
    model.set_weights(random_params(model.layout.creation_order(), seed=1, scale=0.3))
    sched = Scheduler(LR_INIT, LR_MIN, total_step, 'linear')
    return cp, env, model, VecTrainer(env, model, graph=graph), sched


def _em(e, x):
    """device LSTM state -> numpy env-major [B, N, n_h] (feature-major [N, n_h, B] on the tensor-core path)"""
    x = x.detach().cpu().numpy()
    return np.transpose(x, (2, 0, 1)) if e.state_fm else np.swapaxes(x, 0, 1)


def _snap(e, env):
    """The kernel's state at the start of an update (a host copy)."""
    s = dict(params=e.params, ms=e.ms, rng=e.rng, obs0=e.obs_buf[0], fp0=e.fp_buf[0], done0=e.done_buf[0],
             hs=env.hs, vs=env.vs, us=env.us, t=env.t_dev, episode=env.episode_dev)
    s = {k: v.cpu().numpy().copy() for k, v in s.items()}
    s.update(c=_em(e, e.c[e.cur]), h=_em(e, e.h[e.cur]), c_bw=_em(e, e.c_bw), h_bw=_em(e, e.h_bw))
    if e.variant == 'ma2c_dial':
        s['msg'] = np.swapaxes(e.msg[e.cur].cpu().numpy(), 0, 1)
    return s


def _outputs(e):
    """What one update left behind (slots 1..T of the rollout buffers are not touched by the hand-over)."""
    o = dict(obs=e.obs_buf, fp=e.fp_buf, done=e.done_buf, act=e.act_buf, val=e.val_buf, rew=e.rew_buf, grew=e.grew_buf,
             Rs=e.Rs, Advs=e.Advs, R_end=e.R_end, boot_pi=e.boot_pi, boot_act=e.boot_act, grads=e.grads,
             norm=e.norm_out, params=e.params, ms=e.ms, lr=e.lr_dev)
    return {k: v.cpu().numpy().copy() for k, v in o.items()}


def _force_reset(e, env, seed, mask):
    """Restart the envs in mask [B] (float32 device) with the calls `VecTrainer._one_update` makes at an episode end."""
    e.reset_states(mask=mask)
    env.reset_device(mask=mask, obs_out=e.obs_buf[0], fp_out=e.fp_buf[0], philox_seed=seed)
    e.done_buf[0][mask != 0] = 1.0


def _dial_msg(orc_p, h):
    """DIAL's sender-side messages relu(h_j W_mfc_j + b_mfc_j) (oracle/nets.py, OraclePolicy._cell) in float64."""
    N = h.shape[1]
    ht = torch.as_tensor(h, dtype=torch.float64)
    with torch.no_grad():
        return torch.stack([torch.relu(ht[:, j] @ torch.as_tensor(orc_p['dial/mfc_%d/w' % j], dtype=torch.float64) +
                                       torch.as_tensor(orc_p['dial/mfc_%d/b' % j], dtype=torch.float64))
                            for j in range(N)], dim=1).numpy()


def _veh_obs(oenv):
    return np.array([oenv._veh_obs(i) for i in range(oenv.n_agent)])


class _Spy:
    """Records the regime of each rollout and the engine right after each `apply` (before the hand-over's resets)."""

    def __init__(self, e):
        self.saved, self.after_apply = [], []
        roll, apply = e.rollout, e.apply

        def rollout(*a, **k):
            roll(*a, **k)
            self.saved.append(bool(e.saved_rollout))

        def apply_(*a, **k):
            apply(*a, **k)
            s = dict(c=_em(e, e.c[e.cur]), h=_em(e, e.h[e.cur]), c_bw=_em(e, e.c_bw), h_bw=_em(e, e.h_bw),
                     params=e.params.cpu().numpy().copy())
            if e.variant == 'ma2c_dial':
                s['msg'] = np.swapaxes(e.msg[e.cur].cpu().numpy(), 0, 1)
            self.after_apply.append(s)
        e.rollout, e.apply = rollout, apply_


def _near_step(pi, u):
    """distance of u to the nearest interior step of the normalised float64 cdf of pi [..., n_a]"""
    cdf = np.cumsum(pi.astype(np.float64), axis=-1)
    cdf = cdf / cdf[..., -1:]
    return np.abs(cdf[..., :-1] - u[..., None]).min(-1)


@pytest.mark.parametrize('agent,ini,B,fuse,clip', CASES)
def test_training_loop_matches_oracle_update_by_update(agent, ini, B, fuse, clip):
    cp, env, model, vt, sched = _make(agent, ini, B, clip)
    e, lay = model.engine, model.layout
    e.fuse_save = fuse
    N, NH, n_a = e.N, e.n_h, e.n_a
    assert e.T == T and env.T == 3 * T and env.batch_size == T
    assert e.use_tc == (B == 128), 'the env count must select the kernel path under test'
    if e.use_tc:
        assert e.state_fm == (agent != 'ma2c_dial'), 'DIAL keeps env-major state, the others feature-major'
    hp = e.hp
    spy = _Spy(e)
    seed = int(env.seed)
    Pn = N // env.platoon_len
    mask_mat, dist = env.neighbor_mask, env.distance_mask
    forced = np.zeros(B, bool)
    forced[::3] = True

    vt.start()
    # one persistent NumPy env per env, restarted from the same Philox reset draws as the device
    ep_host = np.zeros(B, np.int64)
    oenvs = [OracleCACC(cp['ENV_CONFIG']) for _ in range(B)]

    def restart(idx):
        u = P.reset_uniforms(seed, ep_host, Pn, B)
        for b in idx:
            oenvs[b].reset(u01=u[0, b])
            ep_host[b] += 1
    restart(range(B))

    lrs, norms, resets, worst_ms, worst_msg = [], [], [], 0.0, 0.0
    prev = None
    for k in range(K + 1):
        pre = _snap(e, env)
        # ---- 6. hand-over of update k - 1 (and the start of the run) ------------------------------------------------
        if prev is None:
            reset = np.ones(B, bool)
            assert np.all(pre['c'] == 0) and np.all(pre['h'] == 0)
            assert np.all(pre['done0'] == 1)
        else:
            out, st_boot = prev['out'], prev['st_boot']
            reset = (out['done'][T] != 0) | (forced if k == 1 else False)
            resets.append(reset)
            assert pre['rng'][0] == prev['pre']['rng'][0] and pre['rng'][1] - prev['pre']['rng'][1] == T + 1, \
                ('Philox counter', k, pre['rng'], prev['pre']['rng'])
            keep = ~reset
            assert np.array_equal(pre['obs0'][:, keep], out['obs'][T][:, keep]), ('obs slot 0 != slot T', k)
            assert np.array_equal(pre['fp0'][:, keep], out['fp'][T][:, keep]), ('fp slot 0 != slot T', k)
            assert np.array_equal(pre['done0'][keep], out['done'][T][keep]), ('done slot 0 != slot T', k)
            for n, x in (('c', pre['c']), ('h', pre['h'])):
                ref = st_boot[..., :NH] if n == 'c' else st_boot[..., NH:]
                err = np.abs(x[keep] - ref[keep]).max() if keep.any() else 0.0
                assert err < 1e-5, ('state %s after the bootstrap' % n, k, err)
            for n in ('c', 'h', 'c_bw', 'h_bw'):
                assert np.all(pre[n][reset] == 0), ('%s of a restarted env' % n, k)
            assert np.all(pre['fp0'][:, reset] == np.float32(1.0 / n_a)), ('fingerprint of a restarted env', k)
            assert np.all(pre['done0'][reset] == 1), ('done of a restarted env', k)
            restart(np.where(reset)[0])
            # after apply, before the resets: states_bw := states_fw for every env, DIAL messages under the new weights
            aa = spy.after_apply[k - 1]
            assert np.array_equal(aa['c_bw'], aa['c']) and np.array_equal(aa['h_bw'], aa['h']), ('states_bw after apply', k)
            if agent == 'ma2c_dial':
                # the kernel's own h and weights: only the rounding of one 64-term fp32 dot product separates the cached
                # messages from the float64 ones, while one optimizer step moves them by ~1e-5
                w_new = lay.unpack(out['params'])
                for tag, msg, h in (('after apply', aa['msg'], aa['h']), ('at the start of the update', pre['msg'], pre['h'])):
                    err = np.abs(msg - _dial_msg(w_new, h)).max()
                    worst_msg = max(worst_msg, err)
                    assert err < MSG_TOL, ('DIAL messages ' + tag, k, err)
        np.testing.assert_array_equal(pre['episode'], ep_host, err_msg='episode counters (%d)' % k)
        assert np.array_equal(pre['c_bw'], pre['c']) and np.array_equal(pre['h_bw'], pre['h']), ('states_bw', k)
        for b in range(B):
            o = oenvs[b]
            if reset[b]:
                err = np.abs(pre['obs0'][:, b, :5] - _veh_obs(o)).max()
                assert err < 1e-6, ('obs of a restarted env', k, b, err)
            assert pre['t'][b] == o.t, ('env time', k, b)
            for n, x in (('hs', o.hs_cur), ('vs', o.vs_cur), ('us', o.us_cur)):
                np.testing.assert_allclose(pre[n][:, b], x, rtol=1e-9, atol=1e-12, err_msg='env %s (%d, %d)' % (n, k, b))
        if k == K:
            break

        # ---- the update, then the forced staggering --------------------------------------------------------------------
        vt.update()
        torch.cuda.synchronize()
        e.check_tc()
        out = _outputs(e)
        ls = e.losses()
        if k == 0:
            _force_reset(e, env, vt._seed, torch.as_tensor(forced.astype(np.float32), device=e.device))
        assert spy.saved[k] == (e.use_tc and fuse), ('fused saved rollout', k, spy.saved[k])
        lr = float(np.float32(sched.get(T * B)))
        assert out['lr'][0] == np.float32(lr), ('lr', k, out['lr'][0], lr)
        lrs.append(lr)
        W = lay.unpack(pre['params'])
        obs = [pre['obs0']] + [out['obs'][t] for t in range(1, T + 1)]               # [N, B, 8] per slot
        fps = [pre['fp0']] + [out['fp'][t] for t in range(1, T + 1)]
        dones = np.concatenate([pre['done0'][None], out['done'][1:]])                  # [T + 1, B], pre-step
        obs_o = [oracle_obs(lay, np.swapaxes(obs[t][..., :5], 0, 1).astype(np.float64)) for t in range(T + 1)]
        fp_o = [np.swapaxes(f, 0, 1) for f in fps]                                       # [B, N, n_a]

        # ---- 1. rollout from the kernel's state at the start of the update ------------------------------------------------
        orc = nets.OraclePolicy(agent, model.n_s_ls, n_a, mask_mat, params=W, n_env=B)
        orc.states_fw = torch.tensor(np.concatenate([pre['c'], pre['h']], -1))
        undecided = 0
        for t in range(T + 1):
            pi_o = orc.forward(obs_o[t], dones[t], fp_o[t], None, 'p')                       # [B, N, n_a]
            pi_k = np.swapaxes(out['fp'][t + 1] if t < T else out['boot_pi'], 0, 1)
            err = np.abs(pi_k - pi_o).max()
            assert err < 1e-5, ('pi', k, t, err)
            a_k = (out['act'][t] if t < T else out['boot_act']).T                           # [B, N]
            u = P.action_uniforms(int(pre['rng'][0]), int(pre['rng'][1]) + t, N, B).T      # [B, N]
            np.testing.assert_array_equal(a_k, P.inverse_cdf(pi_k, u, scaled=e.use_tc), err_msg='actions (%d, %d)' % (k, t))
            clear = _near_step(pi_o, u) > 1e-5
            undecided += int((~clear).sum())
            np.testing.assert_array_equal(a_k[clear], P.inverse_cdf(pi_o, u, scaled=e.use_tc)[clear],
                                          err_msg='oracle draws (%d, %d)' % (k, t))
            v_o = orc.forward(obs_o[t], dones[t], fp_o[t], a_k, 'v')                         # [B, N]
            v_k = (out['val'][t] if t < T else out['R_end']).T
            err = np.abs(v_k - v_o).max()
            assert err < 1e-5, ('v' if t < T else 'R_end', k, t, err)
        assert undecided < 1e-3 * (T + 1) * N * B
        st_boot = orc.states_fw.numpy().copy()

        # ---- 2. env: the NumPy envs driven by the kernel's actions -------------------------------------------------------
        for b in range(B):
            o = oenvs[b]
            for t in range(T):
                _, r, done, gr = o.step(out['act'][t, :, b])
                err = np.abs(out['obs'][t + 1][:, b, :5] - _veh_obs(o)).max()
                assert err < 2e-6, ('obs', k, t, b, err)
                assert abs(out['grew'][t, b] - gr) <= 1e-9 * abs(gr) + 1e-12, ('global reward', k, t, b)
                if e.NR > 1:
                    np.testing.assert_allclose(out['rew'][t, :, b], r, rtol=1e-9, atol=1e-12)
                assert float(done) == out['done'][t + 1, b], ('done', k, t, b)

        # ---- 3. returns in float64 -----------------------------------------------------------------------------------
        rn, gamma = float(hp['reward_norm']), float(hp['gamma'])
        for b in range(B):
            r = out['rew'][:, :, b] / rn if e.NR > 1 else np.repeat(out['grew'][:, b:b + 1] / rn, N, 1)
            Re = np.zeros(N) if out['done'][T, b] else out['R_end'][:, b].astype(np.float64)
            oR, oA = nstep_returns(r, out['val'][:, :, b], out['done'][1:, b], Re, gamma, env.coop_gamma, dist)
            err_R, err_A = np.abs(out['Rs'][:, :, b].T - oR).max(), np.abs(out['Advs'][:, :, b].T - oA).max()
            assert err_R < 1e-5 and err_A < 2e-5, ('returns', k, b, err_R, err_A)

        # ---- 4. gradient and losses: float64 autograd from the pre-update weights and states_bw -------------------------------
        o64 = nets.OraclePolicy(agent, model.n_s_ls, n_a, mask_mat, params=W, dtype=torch.float64, n_env=B)
        o64.states_bw = torch.tensor(np.concatenate([pre['c_bw'], pre['h_bw']], -1), dtype=torch.float64)
        mode = RoundoffScale(o64.p)
        with mode:
            summ = o64.backward(obs_o[:T], np.stack(fp_o[:T]).astype(np.float64), np.transpose(out['act'], (0, 2, 1)),
                                dones[:T], np.transpose(out['Rs'], (0, 2, 1)), np.transpose(out['Advs'], (0, 2, 1)), lr,
                                v_coef=hp['v_coef'], e_coef=hp['e_coef'], apply=False)
        g_k = lay.unpack(out['grads'])
        for n in o64.names:
            g64, kink = o64.grads[n].numpy(), mode.K[n].numpy()
            err = np.maximum(np.abs(g_k[n] - g64) - kink, 0).max()
            scale = max(1e-3, np.abs(g64).max())
            assert err <= 2e-5 * scale + 1e-7, ('gradient', k, n, err, scale)
        for n in ('policy_loss', 'value_loss', 'entropy_loss'):
            np.testing.assert_allclose(ls[n], summ[n], rtol=1e-4, atol=1e-5, err_msg='%s (%d)' % (n, k))
        del mode

        # ---- 5. apply: clip + TF-RMSProp (+ consensus) from the kernel's pre-update weights and slots --------------------
        oa = nets.OraclePolicy(agent, model.n_s_ls, n_a, mask_mat, params=W, dtype=torch.float64)
        oa.ms = {n: torch.tensor(v, dtype=torch.float64) for n, v in lay.unpack(pre['ms']).items()}
        oa.grads = o64.grads
        gn = oa.apply_grads(lr, float(hp['max_grad_norm']), float(hp['alpha']), float(hp['epsilon']))
        np.testing.assert_allclose(out['norm'], gn, rtol=2e-4, err_msg='gradient norm (%d)' % k)
        norms.append(np.asarray(gn))
        w_k, ms_k = lay.unpack(out['params']), lay.unpack(out['ms'])
        for n in oa.names:
            np.testing.assert_allclose(w_k[n], oa.p[n].detach().numpy(), rtol=0, atol=3e-6, err_msg='%s (%d)' % (n, k))
            d = float(np.abs(ms_k[n] - oa.ms[n].numpy()).max()) if ms_k[n].size else 0.0
            worst_ms = max(worst_ms, d)
            assert d <= 1e-6, ('RMSProp slot', k, n, d)
        prev = dict(pre=pre, out=out, st_boot=st_boot)

    # ---- the regime this case claims ----------------------------------------------------------------------------------
    assert all(a > b for a, b in zip(lrs, lrs[1:])), ('the lr must change every update', lrs)
    clipped = [bool((g > float(hp['max_grad_norm'])).any()) for g in norms]
    assert all(clipped) if clip else not any(clipped), ('clip regime', clip, [g.max() for g in norms])
    assert any(0 < r.sum() < B for r in resets), 'no hand-over with a mixed reset mask'
    assert np.logical_or.reduce(resets).all(), 'some env was never restarted by a hand-over'
    print('%s B=%d fuse=%d clip=%d: resets per hand-over %s, lr %s, worst |ms - oracle| %.2e, DIAL messages %.2e' % (
        agent, B, fuse, clip, [int(r.sum()) for r in resets], ['%.2e' % x for x in lrs], worst_ms, worst_msg))


def test_graph_replay_matches_eager_update_by_update():
    """NeurComm, tensor cores: a CUDA-graph VecTrainer with the same seeds and the same forced staggering gives the
    eager one's actions, values, gradients, weights, RMSProp slots, Philox counter and env state after every update."""
    B = 128
    runs = []
    for graph in (False, True):
        cp, env, model, vt, _ = _make('ma2c_nc', 'config_ma2c_nc_catchup.ini', B, True, graph=graph)
        e = model.engine
        assert e.use_tc
        vt.start()
        forced = torch.zeros(B, device=e.device)
        forced[::3] = 1
        snaps = []
        for k in range(K):
            vt.update()
            if k == 0:
                _force_reset(e, env, vt._seed, forced)
            torch.cuda.synchronize()
            e.check_tc()
            snaps.append({n: x.clone() for n, x in dict(
                act=e.act_buf, val=e.val_buf, grads=e.grads, params=e.params, ms=e.ms, rng=e.rng, hs=env.hs, vs=env.vs,
                us=env.us, t=env.t_dev, episode=env.episode_dev, done=e.done_buf, obs0=e.obs_buf[0]).items()})
        assert vt.graph is not None if graph else vt.graph is None
        runs.append(snaps)
    for k in range(K):
        for n in runs[0][k]:
            assert torch.equal(runs[0][k][n], runs[1][k][n]), ('graph replay differs from eager', k, n)
    t = runs[0][-1]['t'].cpu().numpy()
    assert len(np.unique(t)) > 1, 'the staggered episodes must be out of step'
