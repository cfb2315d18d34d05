"""GPU: parity of the tensor-core path AT THE SHAPES bench.py TIMES (VERDICT r1, item 1).

For each BASELINE.json configuration, at its per-GPU batch:
  cfg2  config_ma2c_nc_catchup.ini      NeurComm, 8 agents, B = 4096, T = 60   (the headline shape)
  cfg3  config_ma2c_cnet_slowdown.ini   CommNet,  8 agents, B = 512  (4096 envs over 8 GPUs)
  cfg4  config_ma2c_dial_catchup.ini    DIAL,     8 agents, B = 1024 (8192 envs over 8 GPUs)
  cfg5  config_ma2c_nc_grid5x5_stub.ini NeurComm, 25 agents on the 5x5 grid, B = 256, T = 120
one full `rollout` (host uniforms -> pi, sampled actions, v, env step, bootstrap) is replayed step by step through
the batched oracle (oracle/nets.py, fp32 like the reference) on the SAME observations / fingerprints / dones;
the n-step returns are recomputed in float64; then `backward` is compared, tensor by tensor, with the float64
oracle autograd of the recorded batch (accumulated over env chunks -- the loss is a mean over (t, env), so chunk
gradients add up), and `apply` with the oracle's clip + TF-RMSProp step.

Tolerances (north_star): pi, v, returns 1e-5 abs; advantages 2e-5; gradients 2e-5 x max|g| per tensor; weights
3e-6; sampled actions bit-identical to np.random.choice's rule on the kernel's own pi, and equal to the oracle's
choice wherever the uniform is not within 1e-5 of a cdf step; env rows spot-checked against the NumPy env.
"""
import numpy as np
import pytest
import torch

from helpers import load_cfg, random_params
from oracle import nets
from oracle.buffers import nstep_returns
from oracle.cacc import OracleCACC

pytestmark = pytest.mark.gpu

CASES = [('config_ma2c_nc_catchup.ini', 4096, 512),
         ('config_ma2c_cnet_slowdown.ini', 512, 256),
         ('config_ma2c_dial_catchup.ini', 1024, 256),
         ('config_ma2c_nc_grid5x5_stub.ini', 256, 64)]


def _choice(pi, u):
    """np.random.choice(p=pi) given its uniform: searchsorted(cumsum(p64) / sum, u, 'right'); also the distance
    of u to the nearest cdf step (ties are not decidable across implementations)."""
    cdf = np.cumsum(pi.astype(np.float64), axis=-1)
    cdf = cdf / cdf[..., -1:]
    act = np.minimum((cdf <= u[..., None]).sum(-1), pi.shape[-1] - 1)
    return act, np.abs(cdf[..., :-1] - u[..., None]).min(-1)


@pytest.mark.parametrize('ini,B,chunk', CASES)
def test_rollout_backward_apply_at_bench_shape(ini, B, chunk):
    from deeprl_network_b200.agents.engine import PolicyEngine
    from deeprl_network_b200.envs.cacc_env import CACCEnv
    from deeprl_network_b200.layout import ModelLayout
    cp = load_cfg(ini, n_env=B)
    env = CACCEnv(cp['ENV_CONFIG'])
    mc = cp['MODEL_CONFIG']
    agent, N, mask = env.agent, env.n_agent, env.neighbor_mask
    T = mc.getint('batch_size')
    lay = ModelLayout(agent, env.n_s_ls, 4, mask, obs_mode='gather')
    params = random_params(lay.creation_order(), seed=1, scale=0.3)
    hp = dict(v_coef=mc.getfloat('value_coef'), e_coef=mc.getfloat('entropy_coef'), max_grad_norm=mc.getfloat('max_grad_norm'),
              alpha=mc.getfloat('rmsp_alpha'), epsilon=mc.getfloat('rmsp_epsilon'), gamma=mc.getfloat('gamma'),
              reward_norm=mc.getfloat('reward_norm'), reward_clip=mc.getfloat('reward_clip'))
    e = PolicyEngine(lay, B, T, hp, flat_params=lay.pack(params), distance_mask=env.distance_mask,
                     coop_gamma=env.coop_gamma)
    assert e.use_tc, 'this test is about the tensor-core path'
    dev = env.device
    rs = np.random.RandomState(5)
    P = N // env.platoon_len
    u0 = rs.rand(P, B)
    uni = rs.rand(T + 1, N, B)
    env.reset_device(u01=torch.as_tensor(u0).to(dev))
    e.begin_episode(env)
    # a non-trivial recurrent state for half of the envs (done_prev = 0 there): BPTT starts from states_bw != 0
    c0 = (rs.randn(N, B, 64) * 0.5).astype(np.float32)
    h0 = (np.tanh(rs.randn(N, B, 64)) * 0.8).astype(np.float32)
    e.set_states(torch.as_tensor(c0).to(dev), torch.as_tensor(h0).to(dev))
    d0 = (rs.rand(B) < 0.5).astype(np.float32)
    e.done_buf[0].copy_(torch.as_tensor(d0).to(dev))

    e.rollout(env, sample='uniform', uniforms=torch.as_tensor(uni).to(dev))
    assert e.saved_rollout, 'the bench path (rollout p-calls save the BPTT activations) must be the one under test'
    e.compute_returns()
    torch.cuda.synchronize()
    e.check_tc()
    obs = e.obs_buf.cpu().numpy()[..., :5]          # [T+1, N, B, 5]
    fp = e.fp_buf.cpu().numpy()                      # [T+1, N, B, 4]  (slot t+1 = pi of step t)
    dones = e.done_buf.cpu().numpy()                 # [T+1, B]        (slot t = done BEFORE step t)
    acts = e.act_buf.cpu().numpy()                   # [T, N, B]
    vals = e.val_buf.cpu().numpy()
    grew = e.grew_buf.cpu().numpy()                  # [T, B]
    Rs, Advs, R_end = e.Rs.cpu().numpy(), e.Advs.cpu().numpy(), e.R_end.cpu().numpy()
    boot_pi, boot_act = e.boot_pi.cpu().numpy(), e.boot_act.cpu().numpy()

    # ---- 1. rollout: every p-call and v-call against the batched fp32 oracle --------------------------------
    orc = nets.OraclePolicy(agent, env.n_s_ls, 4, mask, params=params, n_env=B)
    st0 = torch.tensor(np.concatenate([np.swapaxes(c0, 0, 1), np.swapaxes(h0, 0, 1)], -1))
    orc.states_fw = st0.clone()
    undecided = 0
    for t in range(T + 1):
        ob_t = [obs[t, i] for i in range(N)]
        fp_t = np.swapaxes(fp[t], 0, 1)
        pi_o = orc.forward(ob_t, dones[t], fp_t, None, 'p')                       # [B, N, 4]
        pi_k = np.swapaxes(fp[t + 1], 0, 1) if t < T else np.swapaxes(boot_pi, 0, 1)
        assert np.abs(pi_k - pi_o).max() < 1e-5, ('pi', t, np.abs(pi_k - pi_o).max())
        a_k = (acts[t] if t < T else boot_act).T                                   # [B, N]
        u_t = uni[t].T
        a_own, _ = _choice(pi_k, u_t)
        np.testing.assert_array_equal(a_k, a_own)
        a_orc, margin = _choice(pi_o, u_t)
        clear = margin > 1e-5
        undecided += int((~clear).sum())
        np.testing.assert_array_equal(a_k[clear], a_orc[clear])
        v_o = orc.forward(ob_t, dones[t], fp_t, a_k, 'v')                         # [B, N]
        v_k = (vals[t] if t < T else R_end).T
        assert np.abs(v_k - v_o).max() < 1e-5, ('v', t, np.abs(v_k - v_o).max())
    assert undecided < 1e-3 * (T + 1) * N * B
    st_k = e.get_states_fw().cpu().numpy()
    assert np.abs(np.swapaxes(st_k, 0, 1) - orc.states_fw.numpy()).max() < 1e-5

    # ---- 2. env rows (chain configs): the NumPy env driven by the kernel's actions ---------------------------
    if env.platoon_len == N:
        for b in list(range(0, B, max(1, B // 12)))[:12]:
            oenv = OracleCACC(cp['ENV_CONFIG'])
            ob = oenv.reset(u01=u0[0, b])
            for t in range(T):
                assert np.abs(np.array(ob) - obs[t, :, b]).max() < 2e-6, ('obs', b, t)
                ob, r, done, gr = oenv.step(acts[t, :, b])
                assert abs(grew[t, b] - gr) <= 1e-9 * abs(gr) + 1e-12
                assert float(done) == dones[t + 1, b]

    # ---- 3. n-step returns / advantages in float64 over the whole batch ---------------------------------------
    assert env.coop_gamma < 0
    gamma, rn = hp['gamma'], hp['reward_norm']
    R = np.where(dones[T][None, :] != 0, 0.0, R_end.astype(np.float64))           # [N, B]
    for t in range(T - 1, -1, -1):
        R = grew[t][None, :] / rn + gamma * R * (1.0 - dones[t + 1][None, :])
        assert np.abs(Rs[t] - R).max() < 1e-5, ('R', t)
        assert np.abs(Advs[t] - (R - vals[t])).max() < 2e-5, ('Adv', t)
    for b in (0, B // 2 + 1, B - 1):                                              # and the oracle's own scan
        Re = np.zeros(N) if dones[T, b] else R_end[:, b]
        oR, oA = nstep_returns(np.repeat(grew[:, b:b + 1] / rn, N, 1), vals[:, :, b], dones[1:, b], Re, gamma)
        assert np.abs(Rs[:, :, b].T - oR).max() < 1e-5 and np.abs(Advs[:, :, b].T - oA).max() < 2e-5

    # ---- 4. backward: float64 oracle autograd, accumulated over env chunks ---------------------------------------
    e.backward()
    torch.cuda.synchronize()
    e.check_tc()
    g_k = lay.unpack(e.grads.cpu().numpy())
    total = None
    for lo in range(0, B, chunk):
        sl = slice(lo, lo + chunk)
        oc = nets.OraclePolicy(agent, env.n_s_ls, 4, mask, params=params, dtype=torch.float64, n_env=chunk)
        oc.states_bw = st0[sl].double().clone()
        obs_t = [[obs[t, i, sl] for i in range(N)] for t in range(T)]
        oc.backward(obs_t, np.transpose(fp[:T, :, sl], (0, 2, 1, 3)), np.transpose(acts[:, :, sl], (0, 2, 1)), dones[:T, sl],
                    np.transpose(Rs[:, :, sl], (0, 2, 1)), np.transpose(Advs[:, :, sl], (0, 2, 1)), 5e-4,
                    v_coef=hp['v_coef'], e_coef=hp['e_coef'], apply=False)
        part = {n: oc.grads[n].numpy() * (chunk / B) for n in oc.names}
        total = part if total is None else {n: total[n] + part[n] for n in part}
        del oc
    rows = []
    for n, ref in total.items():
        err, scale = np.abs(g_k[n] - ref).max(), max(1e-3, np.abs(ref).max())
        rows.append((err / scale, n, err, scale))
    rows.sort(reverse=True)
    print('%s B=%d T=%d: gradient error / max|g| per tensor, worst five: %s' % (
        ini, B, T, ', '.join('%s %.1e' % (n, r) for r, n, _, _ in rows[:5])))
    bad = [(n, err, scale) for r, n, err, scale in rows if err > 2e-5 * scale + 1e-7]
    assert not bad, bad[:8]

    # ---- 5. apply: clip + TF RMSProp on the oracle's gradient vs the kernel's parameters ------------------------
    oa = nets.OraclePolicy(agent, env.n_s_ls, 4, mask, params=params, dtype=torch.float64, n_env=1)
    oa.grads = {n: torch.tensor(total[n]) for n in oa.names}
    norms = oa.apply_grads(5e-4, hp['max_grad_norm'], hp['alpha'], hp['epsilon'])
    e.apply(5e-4)
    torch.cuda.synchronize()
    np.testing.assert_allclose(e.norm_out.cpu().numpy(), norms, rtol=2e-4)
    w = lay.unpack(e.params.cpu().numpy())
    for n in oa.names:
        np.testing.assert_allclose(w[n], oa.p[n].detach().numpy(), rtol=0, atol=3e-6, err_msg=n)
