"""GPU: models of up to 128 agents (NMARL_MAX_AGENT) on every kernel path.

* The device env replays the many-agent reference fixtures (61 and 128 vehicles; tests/golden/make_golden_many_agents.py)
  through the CACCEnv mirror at B = 1, and at a ragged B = 37 whose envs are all reset through `u01` to the reference's
  initial condition.  Tolerances are those of tests/test_gpu_env.py (CUDA's and glibc's float64 cos() may differ by an
  ulp); done flags, collision latches and the -G rewards after a collision are exact.
* All six agents on an 8x8 grid (64 agents) and a 128-vehicle chain run the p / v forward, the backward and two
  clip + RMSProp steps against the float64 oracle (oracle/nets.py), with the per-tensor round-off scale of
  tests/test_gpu_isolated.py (and an allowance for ReLU inputs at 0, see _check_grad): the FP32-FFMA kernels at B = 7 and the tensor-core kernels at B = 128 with both state
  layouts and raw and packed weight-gradient tiles (tc_err == 0).  IA2C / IA2C_FP clip each of their 64 / 128 agents
  separately: norm_out carries one norm per agent.
* `main.py train` then `evaluate` on a 128-vehicle chain (tensor-core path) and an 8x8 grid (FFMA path).
"""
import configparser
import glob
import os

import numpy as np
import pytest
import torch

from gpu_common import HP, bn, check_apply_twice, nb, oracle_obs, to_dev
from helpers import GOLDEN, ROOT, load_cfg, random_params
from oracle import nets

pytestmark = pytest.mark.gpu
FILES = sorted(glob.glob(os.path.join(GOLDEN, 'many*.npz')))
VARIANTS = ['ia2c', 'ia2c_fp', 'ma2c_cu', 'ma2c_nc', 'ma2c_ic3', 'ma2c_dial']
N_A = 4
KINK_UNITS = 2


# ---- environment -------------------------------------------------------------------------------------------------
def _env(g, n_env):
    from deeprl_network_b200.envs.cacc_env import CACCEnv
    cp = load_cfg(str(g['ini']), **eval(str(g['over'])))
    return CACCEnv(cp['ENV_CONFIG'], n_env=n_env)


def _check_step(t, g, obs, rew, grew, done, collided):
    """one env's outputs after step t against the reference"""
    N = int(g['n_vehicle'])
    ref_g = g['ep0_greward'][t]
    assert abs(grew - ref_g) <= 1e-9 * max(1.0, abs(ref_g)), (t, grew, ref_g)
    np.testing.assert_allclose(np.broadcast_to(rew, (N,)), g['ep0_rew'][t], rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(obs.reshape(-1), g['ep0_obs'][t + 1].astype(np.float32), rtol=0, atol=1e-6)
    assert bool(done) == bool(g['ep0_done'][t]), t
    if ref_g == -1000.0 * N:                                  # collision: the -G rewards are exact
        assert collided and grew == ref_g
        np.testing.assert_array_equal(np.broadcast_to(rew, (N,)), g['ep0_rew'][t])


@pytest.mark.parametrize('path', FILES, ids=[os.path.basename(f)[:-4] for f in FILES])
def test_env_replays_many_agent_fixture_b1(path):
    assert len(FILES) == 6
    g = np.load(path, allow_pickle=True)
    env = _env(g, None)
    N = int(g['n_vehicle'])
    assert env.n_agent == N and env.n_env == 1
    if bool(g['test_mode']):
        env.train_mode = True; env.reset(); env.train_mode = False
        ob = env.reset(test_ind=-1)
    else:
        ob = env.reset()
    assert env.seed == int(g['ep0_seed_after'])
    np.testing.assert_array_equal(env.hs[:, 0].cpu().numpy(), g['ep0_h0'])
    np.testing.assert_array_equal(env.vs[:, 0].cpu().numpy(), g['ep0_v0'])
    np.testing.assert_allclose(np.concatenate(ob), g['ep0_obs'][0].astype(np.float32), rtol=0, atol=1e-6)
    n_exact = 0
    for t, a in enumerate(g['ep0_acts']):
        ob, r, d, gr = env.step(a)
        _check_step(t, g, np.concatenate(ob), r, gr, d, env.collision)
        n_exact += int(gr == g['ep0_greward'][t])
    np.testing.assert_allclose(env.hs[:, 0].cpu().numpy(), g['ep0_hs'][-1], rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(env.vs[:, 0].cpu().numpy(), g['ep0_vs_last'], rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(env.us[:, 0].cpu().numpy(), g['ep0_us_last'], rtol=1e-9, atol=1e-9)
    assert n_exact > 0


@pytest.mark.parametrize('path', FILES, ids=[os.path.basename(f)[:-4] for f in FILES])
def test_env_replays_many_agent_fixture_ragged_batch(path):
    """37 envs = one full 32-env block + a ragged one, all reset through u01 to the reference's initial condition"""
    B = 37
    g = np.load(path, allow_pickle=True)
    env = _env(g, B)
    N = int(g['n_vehicle'])
    env.train_mode = not bool(g['test_mode'])
    env.reset_device(u01=torch.full((1, B), float(g['ep0_u01']), dtype=torch.float64, device=env.device))
    np.testing.assert_array_equal(env.hs.cpu().numpy(), np.repeat(g['ep0_h0'][:, None], B, 1))
    np.testing.assert_array_equal(env.vs.cpu().numpy(), np.repeat(g['ep0_v0'][:, None], B, 1))
    for t, a in enumerate(g['ep0_acts']):
        env.step_device(torch.as_tensor(np.repeat(a[:, None], B, 1), dtype=torch.int32, device=env.device))
        obs = env.obs_dev[..., :5].cpu().numpy()
        rew, grew = env.reward_dev.cpu().numpy(), env.greward_dev.cpu().numpy()
        done, col = env.done_dev.cpu().numpy(), env.collision_dev.cpu().numpy()
        for b in range(B):
            _check_step(t, g, obs[:, b], rew[:, b] if rew.shape[0] == N else rew[0, b], grew[b], done[b], bool(col[b]))
        assert np.all(grew == grew[0]) and np.all(rew == rew[:, :1])      # every env ran the same trajectory
    assert np.all(env.t_dev.cpu().numpy() == len(g['ep0_acts']))
    np.testing.assert_allclose(env.hs.cpu().numpy(), np.repeat(g['ep0_hs'][-1][:, None], B, 1), rtol=1e-11, atol=1e-11)


# ---- kernels against the float64 oracle ------------------------------------------------------------------------------
def _mask(shape):
    from deeprl_network_b200.envs.cacc_env import chain_masks, grid_masks
    return grid_masks(8)[0] if shape == 'grid8x8' else chain_masks(128)[0]


def _engine(lay, params, B, T):
    from deeprl_network_b200.agents.engine import PolicyEngine
    eng = PolicyEngine(lay, B, T, dict(HP), flat_params=lay.pack(params))
    assert eng.state_fm == (eng.use_tc and eng.variant != 'ma2c_dial'), 'feature-major state on tensor cores, but DIAL'
    return eng


def _check_grad(tag, n, g, ref):
    """The per-tensor round-off scale of tests/test_gpu_isolated.py, err <= 2e-5 * max(1e-3, max|ref|) + 1e-7, on every
    output unit (last axis) but at most KINK_UNITS of them.  With 128 agents x 128 envs x T steps there are millions of
    encoder ReLU inputs, and a few lie closer to 0 than fp32 round-off: fp32 and fp64 then disagree on whether one row
    reaches one unit, which moves that unit's column of the weight gradient (and its bias) by that row's single
    contribution.  Such a unit is still held to 1e-2 of the tensor's scale; a wrong kernel moves many units."""
    scale = max(1e-3, np.abs(ref).max())
    err = np.abs(g - ref)
    bad = err > 2e-5 * scale + 1e-7
    units = np.unique(np.nonzero(bad)[-1]) if bad.any() else []
    assert len(units) <= KINK_UNITS and err.max() <= 1e-2 * scale, (tag, n, err.max(), scale, len(units))


@pytest.mark.parametrize('B', [7, 128])                                  # 7: FP32 FFMA, 128: tensor cores
@pytest.mark.parametrize('shape', ['grid8x8', 'chain128'])
@pytest.mark.parametrize('variant', VARIANTS)
def test_many_agent_kernels_match_oracle(variant, shape, B):
    from deeprl_network_b200.layout import ModelLayout
    T = 3
    mask = _mask(shape)
    N = len(mask)
    nm = [int(mask[i].sum()) for i in range(N)]
    n_s_ls = {'ia2c': [5 * (1 + k) for k in nm], 'ia2c_fp': [5 * (1 + k) + N_A * k for k in nm]}.get(variant, [5] * N)
    lay = ModelLayout(variant, n_s_ls, N_A, mask, obs_mode='gather')
    params = random_params(lay.creation_order(), seed=11, scale=0.3)
    orc = nets.OraclePolicy(variant, n_s_ls, N_A, mask, params=params, dtype=torch.float64, n_env=B)
    rs = np.random.RandomState(4)
    base = rs.randn(T, B, N, 5).astype(np.float32)
    fp = rs.dirichlet(np.ones(N_A), size=(T, B, N)).astype(np.float32)
    acts = rs.randint(0, N_A, size=(T, B, N))
    dones = np.zeros((T, B), dtype=np.float32); dones[0, ::2] = 1; dones[2, 1::3] = 1
    Rs = rs.randn(T, B, N).astype(np.float32); Advs = rs.randn(T, B, N).astype(np.float32)
    c0 = (rs.randn(B, N, 64) * .5).astype(np.float32); h0 = (rs.rand(B, N, 64) - .5).astype(np.float32)
    st = torch.tensor(np.concatenate([c0, h0], -1), dtype=torch.float64)
    obs_o = [oracle_obs(lay, base[t]) for t in range(T)]
    # oracle: p / v forward of step 0, then the backward from the same states
    orc.states_fw = st.clone()
    pi_o = orc.forward(obs_o[0], dones[0], fp[0].astype(np.float64), None, 'p')
    st_o = orc.states_fw.numpy().copy()
    v_o = orc.forward(obs_o[0], dones[0], fp[0].astype(np.float64), acts[0], 'v')
    orc.states_bw, orc.states_fw = st.clone(), st.clone()
    orc.backward(obs_o, fp.astype(np.float64), acts, dones, Rs, Advs, 5e-4, v_coef=HP['v_coef'], e_coef=HP['e_coef'],
                 apply=False)
    pad = np.ones(lay.n_param, bool)
    for _, o, s in lay.entries:
        pad[o:o + int(np.prod(s))] = False
    tag = '%s %s B=%d' % (variant, shape, B)
    eng = _engine(lay, params, B, T)
    assert eng.use_tc == (B == 128), tag
    # ---- forward p / v ----
    eng.set_states(nb(c0), nb(h0))
    obs_d = torch.zeros(N, B, lay.obs_stride, device='cuda'); obs_d[:, :, :5] = nb(base[0])
    pi_d = torch.zeros(N, B, N_A, device='cuda'); v_d = torch.zeros(N, B, device='cuda')
    eng.step_p(obs_d, nb(fp[0]), to_dev(dones[0]), pi_d)
    np.testing.assert_allclose(bn(pi_d), pi_o, rtol=0, atol=1e-5, err_msg=tag)
    np.testing.assert_allclose(bn(eng.get_states_fw()), st_o, rtol=0, atol=1e-5, err_msg=tag)
    eng.step_v(obs_d, nb(fp[0]), to_dev(dones[0]), nb(acts[0]).int(), v_d)
    np.testing.assert_allclose(bn(v_d), v_o, rtol=0, atol=1e-5, err_msg=tag)
    # ---- backward ----
    eng.T_cur = T
    eng.obs_buf[:T].zero_(); eng.obs_buf[:T, :, :, :5].copy_(to_dev(np.transpose(base, (0, 2, 1, 3))))
    eng.fp_buf[:T].copy_(to_dev(np.transpose(fp, (0, 2, 1, 3))))
    eng.act_buf[:T].copy_(to_dev(np.transpose(acts, (0, 2, 1)), torch.int32))
    eng.done_buf[:T].copy_(to_dev(dones))
    eng.Rs[:T].copy_(to_dev(np.transpose(Rs, (0, 2, 1)))); eng.Advs[:T].copy_(to_dev(np.transpose(Advs, (0, 2, 1))))
    eng.set_states(nb(c0), nb(h0))
    eng.backward()
    torch.cuda.synchronize()
    eng.check_tc()
    flat = eng.grads.cpu().numpy()
    gk = lay.unpack(flat)
    for n in orc.names:
        _check_grad(tag, n, gk[n], orc.grads[n].numpy())
    assert np.all(flat[pad] == 0), tag                        # the layout padding gets exactly zero gradient
    # ---- two optimizer steps; IA2C / IA2C_FP: one norm per agent ----
    assert eng.norm_out.numel() == (N if variant in ('ia2c', 'ia2c_fp') else 1)
    check_apply_twice(eng, orc, lay, pad)
    assert int(eng.tc_err.item()) == 0


# ---- main.py end to end ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('ini,over', [
    ('config_ma2c_nc_catchup.ini', dict(n_vehicle=128, n_env=128)),                  # tensor-core path
    ('config_ia2c_catchup.ini', dict(n_vehicle=64, topology='grid', n_env=7)),      # FP32-FFMA path
], ids=['chain128-ma2c_nc', 'grid8x8-ia2c'])
def test_main_trains_and_evaluates_many_agents(tmp_path, ini, over):
    import main
    cp = configparser.ConfigParser()
    assert cp.read(os.path.join(ROOT, 'config', ini))
    for k, v in over.items():
        cp['ENV_CONFIG'][k] = str(v)
    n_step = cp.getint('MODEL_CONFIG', 'batch_size')
    cp['TRAIN_CONFIG']['total_step'] = str(3 * n_step * over['n_env'])            # three updates
    cp['TRAIN_CONFIG']['log_interval'] = str(n_step * over['n_env'])
    cfg_path = str(tmp_path / 'exp.ini')
    with open(cfg_path, 'w') as f:
        cp.write(f)
    base = str(tmp_path / 'run')
    main.train(main.parse_args(['--base-dir', base, 'train', '--config-dir', cfg_path]))
    rows = open(base + '/data/train_reward.csv').read().strip().split('\n')[1:]
    assert len(rows) == 3
    assert all(np.isfinite(float(r.split(',')[4])) for r in rows)                  # avg_reward
    ckpt = os.listdir(base + '/model')
    assert len(ckpt) == 1 and ckpt[0].startswith('checkpoint-')
    main.evaluate(main.parse_args(['--base-dir', base, 'evaluate', '--evaluation-seeds', '2000']))
    ev = [f for f in os.listdir(base + '/eva_data') if f.endswith('.csv')]
    assert len(ev) == 2, ev                                                         # control + traffic logs
    traffic = [f for f in ev if f.endswith('traffic.csv')][0]
    txt = open(os.path.join(base, 'eva_data', traffic)).read()
    assert 'headway_%d_m' % over['n_vehicle'] in txt
