"""GPU: the device random stream, draw by draw.  Philox is counter-based, so nothing here is statistical: the host
restatement (tests/philox_ref.py, itself held to the published known-answer vectors by tests/test_philox.py) predicts
every sampled action and every reset state exactly -- which agent and env a draw belongs to, which counter each p-call
of a rollout uses, that the counter moves on between rollouts and between replays of a captured graph, and that env
resets draw from their own stream."""
import numpy as np
import pytest
import torch

import philox_ref as P
from gpu_common import HP, ScriptedEnv, bn, make_pair, nb, obs_dev, to_dev
from helpers import load_cfg
from oracle.cacc import OracleCACC
from test_gpu_policy import _inputs
from test_gpu_vec import _make

pytestmark = pytest.mark.gpu
SEED = 0x5EED0BADC0FFEE11                 # both 32-bit halves of the key are in use
CTR0 = (5 << 32) | 0xFFFFFFFE             # the counter's high word matters, and + 3 carries into it


def _expected(eng, pi_dev, counter):
    """actions [N, B] the engine's kernel family draws from its own pi at this counter"""
    u = P.action_uniforms(int(eng.rng[0].item()), counter, eng.N, eng.B)
    return P.inverse_cdf(pi_dev.cpu().numpy(), u, scaled=eng.use_tc)


@pytest.mark.parametrize('offset', [0, 3])
@pytest.mark.parametrize('B', [37, 256])                    # FFMA kernel; tensor-core kernel, two 128-env tiles
@pytest.mark.parametrize('n_a', [2, 4, 7])
@pytest.mark.parametrize('variant', ['ma2c_nc', 'ia2c'])
def test_step_p_draws_the_predicted_actions(variant, n_a, B, offset):
    from deeprl_network_b200 import _lib as L
    eng, _, lay, _ = make_pair(variant, B, n_a=n_a)
    assert eng.use_tc == (B == 256)
    eng.rng.copy_(torch.tensor([SEED, CTR0], dtype=torch.int64))
    rs, base, fp, done, c0, h0 = _inputs(B, seed=4, n_a=n_a)
    obs_d, fp_d, done_d = obs_dev(lay, base), nb(fp), to_dev(done)
    acts = []
    for rep in range(2):                                     # same state, same counter: same draw
        eng.set_states(nb(c0), nb(h0))
        pi_d = torch.zeros(lay.N, B, n_a, device='cuda')
        act_d = torch.full((lay.N, B), -1, dtype=torch.int32, device='cuda')
        eng.step_p(obs_d, fp_d, done_d, pi_d, act_d, L.SAMPLE_PHILOX, rng_offset=offset)
        np.testing.assert_array_equal(act_d.cpu().numpy(), _expected(eng, pi_d, CTR0 + offset))
        acts.append(act_d)
    assert torch.equal(acts[0], acts[1])
    eng.check_tc()
    assert eng.rng.cpu().tolist() == [SEED, CTR0], 'a p-call reads the counter; only nmarl_rng_advance moves it'
    a = acts[0].cpu().numpy()
    assert len(np.unique(a)) == n_a and not np.array_equal(a[0], a[1])      # not one draw shared by a row of agents
    # nmarl_rng_advance: 64-bit add on the counter, the seed stays
    L.check(L.lib().nmarl_rng_advance(L.ptr(eng.rng), (1 << 33) + 5, L.stream()), 'nmarl_rng_advance')
    assert eng.rng.cpu().tolist() == [SEED, CTR0 + (1 << 33) + 5]


@pytest.mark.parametrize('B', [37, 128])                    # 128: the rollout whose p-calls save the BPTT activations
@pytest.mark.parametrize('variant', ['ma2c_nc', 'ma2c_dial'])
def test_rollout_uses_one_counter_per_p_call(variant, B):
    T = 5
    eng, _, lay, _ = make_pair(variant, B, T=T)
    N = lay.N
    rs = np.random.RandomState(8)
    obs = torch.zeros(T + 1, N, B, lay.obs_stride, device='cuda')
    obs[..., :5] = to_dev(rs.randn(T + 1, N, B, 5).astype(np.float32))
    done = to_dev((rs.rand(T + 1, B) < 0.2).astype(np.float32))
    eng.obs_buf[0].copy_(obs[0]); eng.done_buf[0].copy_(done[0])
    seed = int(eng.rng[0].item())
    rollouts = []
    for r in range(2):
        eng.rollout(ScriptedEnv(obs, done), sample='philox', bootstrap=True)
        assert eng.saved_rollout == (B == 128)
        torch.cuda.synchronize()
        eng.check_tc()
        for t in range(T):                                   # fp_buf[t + 1] is the pi the p-call of step t wrote
            np.testing.assert_array_equal(eng.act_buf[t].cpu().numpy(), _expected(eng, eng.fp_buf[t + 1], r * (T + 1) + t),
                                          err_msg='rollout %d step %d' % (r, t))
        np.testing.assert_array_equal(eng.boot_act.cpu().numpy(), _expected(eng, eng.boot_pi, r * (T + 1) + T),
                                      err_msg='rollout %d bootstrap' % r)
        assert eng.rng.cpu().tolist() == [seed, (r + 1) * (T + 1)]
        rollouts.append(eng.act_buf.clone())
        eng.saved_rollout = False
        eng.roll_buffers()
    assert not torch.equal(rollouts[0], rollouts[1])


def test_graph_replays_draw_fresh_predicted_actions():
    """VecTrainer(graph=True) at B = 128: update k, eager or replayed from the captured graph, uses counters
    k * (T + 1) + t -- the counter lives on the device and nmarl_rng_advance is part of the graph."""
    cp, env, model, vt = _make('ma2c_nc', 128, graph=True, sample='philox')
    e = model.engine
    assert e.use_tc
    T, seed = e.T, int(e.rng[0].item())
    vt.start()
    seen = []
    for k in range(3):
        vt.update()
        torch.cuda.synchronize()
        e.check_tc()
        assert (vt.graph is not None) and e.rng.cpu().tolist() == [seed, (k + 1) * (T + 1)]
        for t in range(T):
            np.testing.assert_array_equal(e.act_buf[t].cpu().numpy(), _expected(e, e.fp_buf[t + 1], k * (T + 1) + t),
                                          err_msg='update %d step %d' % (k, t))
        np.testing.assert_array_equal(e.boot_act.cpu().numpy(), _expected(e, e.boot_pi, k * (T + 1) + T))
        seen.append(e.act_buf.clone())
    assert not torch.equal(seen[1], seen[2])                # two replays of the same graph


@pytest.mark.parametrize('bit', [0, 40])
def test_seed_bits_reach_the_draws(bit):
    from deeprl_network_b200 import _lib as L
    from deeprl_network_b200.agents.engine import PolicyEngine
    B = 37
    _, _, lay, params = make_pair('ma2c_nc', B)
    rs, base, fp, done, c0, h0 = _inputs(B, seed=4)
    out = []
    for seed in (1234, 1234, 1234 ^ (1 << bit)):
        eng = PolicyEngine(lay, B, 4, dict(HP), flat_params=lay.pack(params), rng_seed=seed)
        assert eng.rng.cpu().tolist() == [seed, 0]
        pi_d = torch.zeros(lay.N, B, 4, device='cuda'); act_d = torch.zeros(lay.N, B, dtype=torch.int32, device='cuda')
        eng.step_p(obs_dev(lay, base), nb(fp), to_dev(done), pi_d, act_d, L.SAMPLE_PHILOX)
        np.testing.assert_array_equal(act_d.cpu().numpy(), _expected(eng, pi_d, 0))
        out.append(act_d)
    assert torch.equal(out[0], out[1]) and not torch.equal(out[0], out[2])


@pytest.mark.parametrize('cfg,n_platoon', [('config_ma2c_nc_catchup.ini', 1), ('config_ma2c_nc_slowdown.ini', 1),
                                           ('config_ma2c_nc_grid5x5_stub.ini', 5)])
def test_env_reset_draws_the_predicted_state(cfg, n_platoon):
    """reset_device without host uniforms: env b, platoon p starts from OracleCACC.reset(u01 = the reset stream's draw for
    (seed, episode of env b, p, b)), bit for bit; a masked reset moves only the masked envs on to their next episode."""
    from deeprl_network_b200.envs.cacc_env import CACCEnv
    B, seed = 37, (0xABCD << 32) | 77
    env = CACCEnv(load_cfg(cfg)['ENV_CONFIG'], n_env=B)
    N, Lp = env.n_agent, env.n_agent // n_platoon
    orc = OracleCACC(load_cfg(cfg, n_vehicle=Lp)['ENV_CONFIG'])

    def check(episode):
        u = P.reset_uniforms(seed, episode, n_platoon, B)
        hs, vs = env.hs.cpu().numpy(), env.vs.cpu().numpy()
        for b in range(B):
            for p in range(n_platoon):
                orc.reset(u01=u[p, b])
                np.testing.assert_array_equal(hs[p * Lp:(p + 1) * Lp, b], orc.hs_cur, err_msg='env %d platoon %d' % (b, p))
                np.testing.assert_array_equal(vs[p * Lp:(p + 1) * Lp, b], orc.vs_cur, err_msg='env %d platoon %d' % (b, p))
                assert env.v_init[p, b].item() == orc.v0s[0]
        return u

    env.reset_device(u01=None, philox_seed=seed)
    u0 = check(np.zeros(B, dtype=int))
    assert len(np.unique(u0)) == u0.size
    mask = torch.zeros(B, device=env.device); mask[1::3] = 1
    env.reset_device(u01=None, mask=mask, philox_seed=seed)
    episode = np.zeros(B, dtype=int); episode[1::3] = 1
    u1 = check(episode)
    assert np.all(u1[:, 1::3] != u0[:, 1::3]) and np.array_equal(u1[:, ::3], u0[:, ::3])
    np.testing.assert_array_equal(env.episode_dev.cpu().numpy(), episode + 1)
