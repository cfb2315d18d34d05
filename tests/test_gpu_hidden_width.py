"""GPU: LSTM widths num_lstm = 16 and 32 on the FP32-FFMA kernels (the tensor-core kernels are built for 64 only).

* All six agents on the 8-agent chain run the p / v forward, the backward (T = 8, dones inside the batch) and two
  clip + RMSProp steps against the float64 oracle (oracle/nets.py) at B = 7 and B = 128.  B = 128 would take the
  tensor-core path at width 64; at 16 / 32 the engine must stay on the FFMA kernels.  ma2c_cu's optimizer step runs
  the consensus update, so check_apply_twice covers nmarl_consensus_update at these widths.
* Heterogeneous NeurComm and DIAL with an isolated agent at width 32.
* Drop-in replay of the fixtures recorded from the UNMODIFIED reference at these widths
  (tests/golden/make_golden_hidden.py, replayed by the oracle in tests/test_hidden_width_parity.py): the six
  tfnet_h{16,32}_<agent> through main.init_agent + Trainer (as tests/test_gpu_tfnet.py), and hetero_h32_ma2c_nc /
  hetero_h32_ia2c_fp -- heterogeneous agents, the last one without neighbours -- through the public classes at B = 1
  (as tests/test_gpu_hetero.py / tests/test_gpu_hetero_ia2c.py).  Initial weights exact, pi / v / R within 1e-5,
  logged rewards within rtol 1e-6, the sampled trained weights within 2e-5, the embedding padding still exactly 0.
* VecTrainer: a captured CUDA graph replays three updates bit for bit like eager execution.
* `main.py train` then `evaluate` from an .ini with num_lstm = 32; the checkpoint holds the reference's shapes.
* C ABI: a descriptor whose s_dim gives n_h = 48 is refused with a message; a packed-operand buffer passed at
  n_h = 32 is ignored (same outputs as without it).
"""
import configparser
import contextlib
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch

from gpu_common import HP, bn, check_apply_twice, nb, oracle_obs, to_dev
from helpers import ROOT, golden, load_cfg, random_params
from oracle import nets
from oracle.cacc import chain_masks
from test_gpu_hetero import _padding as hetero_padding
from test_hetero_ia2c_parity import replay_agent
from test_hetero_parity import replay, w1_error
from test_hidden_width_parity import TFNET_H, width_cfg
from test_tfnet_parity import Rec

pytestmark = pytest.mark.gpu
VARIANTS = ['ia2c', 'ia2c_fp', 'ma2c_cu', 'ma2c_nc', 'ma2c_ic3', 'ma2c_dial']
N_A = 4


def _layout(variant, n_h, mask):
    from deeprl_network_b200.layout import ModelLayout
    nm = [int(mask[i].sum()) for i in range(len(mask))]
    n_s_ls = {'ia2c': [5 * (1 + k) for k in nm], 'ia2c_fp': [5 * (1 + k) + N_A * k for k in nm]}.get(variant, [5] * len(mask))
    return ModelLayout(variant, n_s_ls, N_A, mask, n_h=n_h, n_fc=n_h, obs_mode='gather'), n_s_ls


def _padding(lay, names):
    pad = np.ones(lay.n_param, bool)
    for n in names:
        if hasattr(lay, '_idx'):
            pad[lay._idx[n]] = False
        else:
            o, s = lay.by_name[n]
            pad[o:o + int(np.prod(s))] = False
    if hasattr(lay, 'pi_pad'):
        pad[lay.pi_pad] = False
    return pad


def _check_grads(tag, gk, orc):
    for n in orc.names:
        ref = orc.grads[n].numpy()
        err, scale = np.abs(gk[n] - ref).max(), max(1e-3, np.abs(ref).max())
        assert err <= 2e-5 * scale + 1e-7, (tag, n, err, scale)


def _run_against_oracle(tag, eng, orc, lay, n_h, obs_o, base_dev, fp, acts, dones, Rs, Advs, advs_kernel=None, judge=None):
    """p / v forward of step 0, backward over T steps, gradients, padding and two optimizer steps.  `judge` replaces
    the per-tensor gradient check: judge.mode(orc) is active around the oracle's backward, then
    judge.check(tag, kernel gradients, orc) (tests/test_gpu_narrow_widths.py)."""
    T, B, N = acts.shape
    rs = np.random.RandomState(5)
    c0 = (rs.randn(B, N, n_h) * .5).astype(np.float32); h0 = (rs.rand(B, N, n_h) - .5).astype(np.float32)
    st = torch.tensor(np.concatenate([c0, h0], -1), dtype=torch.float64)
    n_a = fp.shape[-1]
    # ---- forward p / v ----
    orc.states_fw = st.clone()
    pi_o = orc.forward(obs_o[0], dones[0], fp[0].astype(np.float64), None, 'p')
    st_o = orc.states_fw.numpy().copy()
    v_o = orc.forward(obs_o[0], dones[0], fp[0].astype(np.float64), acts[0], 'v')
    eng.set_states(nb(c0), nb(h0))
    pi_d = torch.zeros(N, B, n_a, device='cuda'); v_d = torch.zeros(N, B, device='cuda')
    eng.step_p(base_dev[0], nb(fp[0]), to_dev(dones[0]), pi_d)
    pk = bn(pi_d)
    if isinstance(pi_o, list):                               # heterogeneous: one [B, n_a_i] array per agent
        for i in range(N):
            w = np.asarray(pi_o[i]).shape[-1]
            np.testing.assert_allclose(pk[:, i, :w], pi_o[i], rtol=0, atol=1e-5, err_msg=tag)
            assert np.all(pk[:, i, w:] == 0), tag
    else:
        np.testing.assert_allclose(pk, pi_o, rtol=0, atol=1e-5, err_msg=tag)
    np.testing.assert_allclose(bn(eng.get_states_fw()), st_o, rtol=0, atol=1e-5, err_msg=tag)
    eng.step_v(base_dev[0], nb(fp[0]), to_dev(dones[0]), nb(acts[0]).int(), v_d)
    np.testing.assert_allclose(bn(v_d), v_o, rtol=0, atol=1e-5, err_msg=tag)
    # ---- backward ----
    orc.states_bw, orc.states_fw = st.clone(), st.clone()
    with judge.mode(orc) if judge else contextlib.nullcontext():
        summ = orc.backward(obs_o, fp.astype(np.float64), acts, dones, Rs, Advs, 5e-4, v_coef=HP['v_coef'],
                            e_coef=HP['e_coef'], apply=False)
    eng.T_cur = T
    eng.obs_buf[:T].copy_(base_dev)
    eng.fp_buf[:T].copy_(to_dev(np.transpose(fp, (0, 2, 1, 3))))
    eng.act_buf[:T].copy_(to_dev(np.transpose(acts, (0, 2, 1)), torch.int32))
    eng.done_buf[:T].copy_(to_dev(dones))
    eng.Rs[:T].copy_(to_dev(np.transpose(Rs, (0, 2, 1))))
    eng.Advs[:T].copy_(to_dev(np.transpose(Advs if advs_kernel is None else advs_kernel, (0, 2, 1))))
    eng.set_states(nb(c0), nb(h0))
    eng.backward()
    torch.cuda.synchronize()
    flat = eng.grads.cpu().numpy()
    (judge.check if judge else _check_grads)(tag, lay.unpack(flat), orc)
    losses = eng.losses()
    for k in ('policy_loss', 'value_loss', 'entropy_loss'):        # per agent, the reference's weighting
        ref = np.asarray(summ[k], dtype=np.float64).ravel()
        np.testing.assert_allclose(losses[k], ref, rtol=0, atol=1e-5 * max(1.0, np.abs(ref).max()), err_msg=tag + ' ' + k)
    pad = _padding(lay, orc.names)
    assert np.all(flat[pad] == 0), tag                        # the layout padding gets exactly zero gradient
    check_apply_twice(eng, orc, lay, pad)


@pytest.mark.parametrize('B', [7, 128])
@pytest.mark.parametrize('n_h', [16, 32])
@pytest.mark.parametrize('variant', VARIANTS)
def test_narrow_kernels_match_oracle(variant, n_h, B):
    from deeprl_network_b200.agents.engine import PolicyEngine
    T = 8
    mask, _ = chain_masks(8)
    N = len(mask)
    lay, n_s_ls = _layout(variant, n_h, mask)
    params = random_params(lay.creation_order(), seed=3, scale=0.3)
    orc = nets.OraclePolicy(variant, n_s_ls, N_A, mask, n_h=n_h, n_fc=n_h, params=params, dtype=torch.float64, n_env=B)
    eng = PolicyEngine(lay, B, T, dict(HP), flat_params=lay.pack(params))
    assert eng.use_tc is False and eng.wpack is None
    assert eng.c[0].shape == (N, B, n_h)
    rs = np.random.RandomState(4)
    base = rs.randn(T, B, N, 5).astype(np.float32)
    fp = rs.dirichlet(np.ones(N_A), size=(T, B, N)).astype(np.float32)
    acts = rs.randint(0, N_A, size=(T, B, N))
    dones = np.zeros((T, B), dtype=np.float32); dones[0, ::2] = 1; dones[4, 1::3] = 1
    Rs = rs.randn(T, B, N).astype(np.float32); Advs = rs.randn(T, B, N).astype(np.float32)
    obs_o = [oracle_obs(lay, base[t]) for t in range(T)]
    base_dev = torch.zeros(T, N, B, lay.obs_stride, device='cuda')
    base_dev[..., :5] = to_dev(np.transpose(base, (0, 2, 1, 3)))
    _run_against_oracle('%s n_h=%d B=%d' % (variant, n_h, B), eng, orc, lay, n_h, obs_o, base_dev, fp, acts, dones,
                        Rs, Advs)
    assert eng.norm_out.numel() == (N if variant in ('ia2c', 'ia2c_fp') else 1)


@pytest.mark.parametrize('name', ['hetero_iso_ma2c_nc', 'hetero_iso_ma2c_dial'])
def test_narrow_hetero_isolated_agent_matches_oracle(name):
    """width 32, heterogeneous agents, the last agent without neighbours (no message / fingerprint encoder)"""
    from deeprl_network_b200.agents.engine import PolicyEngine
    from deeprl_network_b200.layout import HeteroLayout
    n_h, B, T = 32, 7, 8
    agent = name[len('hetero_iso_'):]
    g = golden(name)
    n_s, n_a, mask = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']], g['mask']
    N = len(n_s)
    assert min(int(mask[i].sum()) for i in range(N)) == 0
    lay = HeteroLayout(agent, n_s, n_a, mask, n_h=n_h, n_fc=n_h)
    params = random_params(lay.creation_order(), seed=2, scale=0.3)
    orc = nets.OraclePolicy(agent, n_s, n_a, mask, n_h=n_h, n_fc=n_h, params=params, dtype=torch.float64, n_env=B)
    eng = PolicyEngine(lay, B, T, dict(HP), flat_params=lay.pack(params))
    rs = np.random.RandomState(1)
    ob = rs.randn(T, B, N, max(n_s)).astype(np.float32)
    fp = np.zeros((T, B, N, max(n_a)), dtype=np.float32)
    for i in range(N):
        ob[..., i, n_s[i]:] = 0
        fp[..., i, :n_a[i]] = rs.dirichlet(np.ones(n_a[i]), size=(T, B))
    acts = np.stack([rs.randint(0, n_a[i], size=(T, B)) for i in range(N)], axis=-1)
    dones = np.zeros((T, B), dtype=np.float32); dones[0, ::2] = 1; dones[5, 1::2] = 1
    Rs = rs.randn(T, B, N).astype(np.float32); Advs = rs.randn(T, B, N).astype(np.float32)
    obs_o = [[ob[t][:, i, :n_s[i]] for i in range(N)] for t in range(T)]
    base_dev = torch.zeros(T, N, B, lay.obs_stride, device='cuda')
    base_dev[..., :max(n_s)] = to_dev(np.transpose(ob, (0, 2, 1, 3)))
    # quirk Q7: the kernels get the advantages summed over agents (engine.compute_returns)
    _run_against_oracle(name, eng, orc, lay, n_h, obs_o, base_dev, fp, acts, dones, Rs, Advs,
                        advs_kernel=np.repeat(Advs.sum(-1, keepdims=True), N, -1))


def _vec(agent, n_h, B, graph):
    from deeprl_network_b200.agents.models import MA2C_DIAL, MA2C_NC
    from deeprl_network_b200.envs.cacc_env import CACCEnv
    from deeprl_network_b200.utils import VecTrainer
    cp = load_cfg({'ma2c_nc': 'config_ma2c_nc_catchup.ini', 'ma2c_dial': 'config_ma2c_dial_catchup.ini'}[agent], n_env=B)
    cp['MODEL_CONFIG']['num_lstm'] = str(n_h)
    env = CACCEnv(cp['ENV_CONFIG'])
    cls = {'ma2c_nc': MA2C_NC, 'ma2c_dial': MA2C_DIAL}[agent]
    model = cls(env.n_s_ls, env.n_a_ls, env.neighbor_mask, env.distance_mask, env.coop_gamma, 10 ** 6,
                cp['MODEL_CONFIG'], seed=12, n_env=B)
    return env, model, VecTrainer(env, model, graph=graph)


@pytest.mark.parametrize('n_h', [16, 32])
@pytest.mark.parametrize('agent', ['ma2c_nc', 'ma2c_dial'])
def test_narrow_graph_replay_equals_eager(agent, n_h):
    outs = []
    for graph in (False, True):
        env, model, vt = _vec(agent, n_h, 256, graph)
        assert model.layout.n_h == n_h and model.engine.use_tc is False
        vt.start()
        for _ in range(3):
            vt.update()
        torch.cuda.synchronize()
        outs.append((model.engine.params.clone(), model.engine.grew_buf.clone()))
    assert torch.isfinite(outs[0][0]).all()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize('n_env', [1, 128])
def test_main_trains_and_evaluates_width_32(tmp_path, n_env):
    import main
    from oracle.nets import param_shapes
    cp = configparser.ConfigParser()
    assert cp.read(os.path.join(ROOT, 'config', 'config_ma2c_nc_catchup.ini'))
    cp['MODEL_CONFIG']['num_lstm'] = '32'
    cp['ENV_CONFIG']['n_env'] = str(n_env)
    n_step = cp.getint('MODEL_CONFIG', 'batch_size')
    cp['TRAIN_CONFIG']['total_step'] = str(3 * n_step * n_env)
    cp['TRAIN_CONFIG']['log_interval'] = str(n_step * n_env)
    cfg_path = str(tmp_path / 'exp.ini')
    with open(cfg_path, 'w') as f:
        cp.write(f)
    base = str(tmp_path / 'run')
    main.train(main.parse_args(['--base-dir', base, 'train', '--config-dir', cfg_path]))
    ckpt = os.listdir(base + '/model')
    assert len(ckpt) == 1 and ckpt[0].startswith('checkpoint-')
    main.evaluate(main.parse_args(['--base-dir', base, 'evaluate', '--evaluation-seeds', '2000']))
    assert len([f for f in os.listdir(base + '/eva_data') if f.endswith('.csv')]) == 2
    # a fresh model of the same config loads the checkpoint; its weights have the reference's names and shapes
    env = main.init_env(cp['ENV_CONFIG'])
    model = main.init_agent(env, cp['MODEL_CONFIG'], 10 ** 6, 12)
    assert model.load(base + '/model/')
    w = model.get_weights()
    want = param_shapes('ma2c_nc', env.n_s_ls, env.n_a, env.neighbor_mask, n_h=32, n_fc=32)
    want = dict(want.items() if isinstance(want, dict) else want)
    assert {k: tuple(v.shape) for k, v in w.items()} == {k: tuple(s) for k, s in want.items()}
    assert w['nc/lstm_comm_0/wx_hid'].shape == (96, 128)
    assert all(np.all(np.isfinite(v)) for v in w.values())


def test_abi_width_checks_and_ignored_wpack():
    from deeprl_network_b200 import _lib as L
    from deeprl_network_b200.agents.engine import PolicyEngine
    mask, _ = chain_masks(8)
    lay, _ = _layout('ma2c_nc', 32, mask)
    params = lay.pack(random_params(lay.creation_order(), seed=7))
    B, T, N = 128, 4, 8
    rs = np.random.RandomState(0)
    obs = torch.zeros(N, B, lay.obs_stride, device='cuda'); obs[..., :5] = to_dev(rs.randn(N, B, 5))
    fp = to_dev(rs.dirichlet(np.ones(N_A), size=(N, B)))
    done = to_dev((rs.rand(B) < 0.3).astype(np.float32))
    # n_h = 48 (NeurComm s_dim = 3 * 48) has no kernel: the call fails with a message
    bad = PolicyEngine(lay, B, T, dict(HP), flat_params=params)
    bad.model.s_dim = 3 * 48
    with pytest.raises(RuntimeError, match='n_h 48'):
        bad.step_p(obs, fp, done, torch.zeros(N, B, N_A, device='cuda'))
    # the tensor-core operands exist for n_h = 64 only
    wp = torch.zeros(max(lay.n_wp, 4), device='cuda')
    good = PolicyEngine(lay, B, T, dict(HP), flat_params=params)
    assert L.lib().nmarl_pack_weights(ctypes.byref(good.model), L.ptr(good.params), L.ptr(good.wt), L.ptr(wp), L.stream()) != 0
    assert 'n_h' in L.lib().nmarl_last_error().decode()
    Rs, Advs = to_dev(rs.randn(T, N, B)), to_dev(rs.randn(T, N, B))
    # a packed-operand buffer at n_h = 32 is ignored: the FFMA kernels run and give the same bits as wpack = NULL
    outs = []
    for with_wpack in (False, True):
        eng = PolicyEngine(lay, B, T, dict(HP), flat_params=params)
        if with_wpack:
            eng.wpack = wp
        eng.set_states(torch.zeros(N, B, 32, device='cuda'), torch.zeros(N, B, 32, device='cuda'))
        pi = torch.zeros(N, B, N_A, device='cuda')
        eng.step_p(obs, fp, done, pi)
        v = torch.zeros(N, B, device='cuda')
        eng.step_v(obs, fp, done, torch.zeros(N, B, dtype=torch.int32, device='cuda'), v)
        eng.T_cur = T
        eng.obs_buf[:T].copy_(obs); eng.fp_buf[:T].copy_(fp); eng.done_buf[:T].copy_(done)
        eng.Rs.copy_(Rs); eng.Advs.copy_(Advs)
        eng.backward()
        torch.cuda.synchronize()
        outs.append((pi.clone(), v.clone(), eng.get_states_fw().clone(), eng.grads.clone()))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize('name', TFNET_H)
def test_drop_in_path_follows_reference_at_narrow_width(name):
    import main
    from deeprl_network_b200.envs.cacc_env import CACCEnv
    from deeprl_network_b200.utils import Counter, Trainer
    g = golden(name)
    n_h = int(g['n_h'])
    cp = width_cfg(str(g['ini']), n_h)
    env = CACCEnv(cp['ENV_CONFIG'])
    model = main.init_agent(env, cp['MODEL_CONFIG'], 10 ** 6, 12)
    assert model.layout.n_h == n_h and model.engine.use_tc is False
    w0 = model.get_weights()
    names = [str(x) for x in g['names']]
    for n in names:
        assert hashlib.sha256(np.ascontiguousarray(w0[n]).tobytes()).hexdigest() == str(g['w0sha/' + n]), n
    rec = Rec(model)
    counter = Counter(int(g['total_step']), 10 ** 9, 10 ** 9)
    tr = Trainer(env, rec, counter, None)
    tr.run()
    assert counter.cur_step == int(g['cur_step']) and env.seed == int(g['seed_after'])
    trace = np.concatenate(rec.log)
    assert trace.shape == g['trace'].shape
    assert np.abs(trace - g['trace']).max() < 1e-5
    got = np.array([[d['step'], d['avg_reward'], d['std_reward']] for d in tr.data])
    np.testing.assert_allclose(got, g['data'], rtol=1e-6)
    w1 = model.get_weights()
    for n in names:
        assert w1_error(g, n, w1[n]) < 2e-5, n


@pytest.mark.parametrize('name', ['hetero_h32_ma2c_nc', 'hetero_h32_ia2c_fp'])
def test_drop_in_hetero_follows_reference_at_width_32(name):
    from deeprl_network_b200.agents.models import IA2C_FP, MA2C_NC
    agent, g = name[len('hetero_h32_'):], golden(name)
    mc = width_cfg('config_ma2c_nc_catchup.ini', 32)['MODEL_CONFIG']
    mc['batch_size'] = str(int(g['n_step']))
    n_s, n_a = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']]
    assert min(int(g['mask'][i].sum()) for i in range(len(n_s))) == 0          # an agent without neighbours
    np.random.seed(12)
    m = {'ma2c_nc': MA2C_NC, 'ia2c_fp': IA2C_FP}[agent](n_s, n_a, g['mask'], np.zeros_like(g['mask']), -1.0, 10 ** 6,
                                                       mc, seed=12)
    assert not m.identical_agent and m.layout.n_h == 32
    w0 = m.get_weights()
    names = [str(n) for n in g['names']]
    assert names == [n for n, _ in m.layout.creation_order()]
    for n in names:
        assert hashlib.sha256(np.ascontiguousarray(w0[n]).tobytes()).hexdigest() == str(g['w0sha/' + n]), n
    m.reset()
    if agent == 'ma2c_nc':
        trace = replay(g, lambda ob, d, fp: m.forward(ob, d, fp), lambda ob, d, fp, a: m.forward(ob, d, fp, a, 'v'),
                       m.add_transition, lambda R: m.backward(R, 0))
    else:
        trace = replay_agent(g, agent, m)
    assert trace.shape == g['trace'].shape
    assert np.abs(trace - g['trace']).max() < 1e-5
    w1 = m.get_weights()
    for n in names:
        assert w1_error(g, n, w1[n]) < 2e-5, n
    flat = m.engine.params.cpu().numpy()
    assert np.all(flat[m.layout.pi_pad] == np.float32(-1e30))
    assert np.all(flat[hetero_padding(m.layout)] == 0)
