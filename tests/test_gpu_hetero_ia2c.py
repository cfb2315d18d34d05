"""GPU: heterogeneous IA2C / IA2C_FP / IA2C_CU on the CUDA path.

(1) Drop-in (B = 1): the public IA2C / IA2C_FP / IA2C_CU classes replay the scripted stream of
    tests/golden/hetero_{,iso_,iso0_}{ia2c,ia2c_fp,ma2c_cu}.npz -- recorded from the UNMODIFIED reference classes with
    n_s = [5,7,4,6,5,3], n_a = [4,3,5,2,4,3] on the TF shim -- through their reference signatures (IA2C_FP with the
    neighbours' policies appended to every observation), from the same NumPy-stream initial weights (exact): every
    pi / v / R within 1e-5, the sampled trained weights within 2e-5, and after the three updates every padding float of
    the embedding is still exactly 0 (the padded actions' -1e30 biases unchanged).
(2) Batched kernels against the float64 oracle (tests/hetero_ia2c_oracle.py): B = 7 (FP32-FFMA), B = 128 and
    B = 256 (tensor cores: one and two 128-env tiles per agent, feature-major state, tc_err == 0).  States, loss terms and every gradient entry are
    judged with the round-off scale of tests/test_gpu_tc_paths.py, the padding gets exactly zero gradient; then two
    optimizer steps: per-group norm_out, the weights and the untouched padding.
(3) IA2C_CU: nmarl_consensus_update alone (zero gradients) gives the oracle's consensus_update of the LSTM blocks and
    leaves everything else bit for bit."""
import hashlib

import numpy as np
import pytest
import torch

from gpu_common import HP, check_apply_twice, nb, to_dev
from helpers import golden, load_cfg, random_params
from hetero_ia2c_oracle import HeteroIA2COracle
from test_gpu_hetero import _padding
from test_gpu_tc_paths import FLOOR, NH, RoundoffScale, _check, _engine, _inputs, _result, _states, _used
from test_hetero_ia2c_parity import GOLDEN, replay_agent, variant_of
from test_hetero_parity import w1_error

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('name', GOLDEN)
def test_drop_in_hetero_ia2c_follows_reference_golden(name):
    from deeprl_network_b200.agents.models import IA2C, IA2C_CU, IA2C_FP
    agent, g = variant_of(name), golden(name)
    mc = load_cfg('config_ma2c_nc_catchup.ini')['MODEL_CONFIG']
    mc['batch_size'] = str(int(g['n_step']))
    n_s, n_a = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']]
    cls = {'ia2c': IA2C, 'ia2c_fp': IA2C_FP, 'ma2c_cu': IA2C_CU}[agent]
    np.random.seed(12)
    m = cls(n_s, n_a, g['mask'], np.zeros_like(g['mask']), -1.0, 10 ** 6, mc, seed=12)
    assert not m.identical_agent
    w0 = m.get_weights()
    names = [str(n) for n in g['names']]
    assert names == [n for n, _ in m.layout.creation_order()]
    for n in names:
        assert hashlib.sha256(np.ascontiguousarray(w0[n]).tobytes()).hexdigest() == str(g['w0sha/' + n]), n
    m.reset()
    trace = replay_agent(g, agent, m)
    assert trace.shape == g['trace'].shape             # the policies come back at each agent's own width
    assert np.abs(trace - g['trace']).max() < 1e-5
    w1 = m.get_weights()
    for n in names:
        assert w1_error(g, n, w1[n]) < 2e-5, n
    flat = m.engine.params.cpu().numpy()
    assert np.all(flat[m.layout.pi_pad] == np.float32(-1e30))
    assert np.all(flat[_padding(m.layout)] == 0)


def _setup(name, B, T=4):
    from deeprl_network_b200.layout import HeteroLayout
    agent, g = variant_of(name), golden(name)
    n_s, n_a, mask = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']], g['mask']
    lay = HeteroLayout(agent, n_s, n_a, mask)
    params = random_params(lay.creation_order(), seed=2, scale=0.3)
    c = dict(B=B, T=T, dones='mixed')
    return agent, lay, params, c, n_s, n_a


def _kernel_advs(agent, Advs):
    # IA2C_CU: the kernels get the advantages summed over agents (quirk Q7, engine.compute_returns); IA2C / IA2C_FP
    # have one loss per agent and get their own
    return np.repeat(Advs.sum(-1, keepdims=True), Advs.shape[-1], -1) if agent == 'ma2c_cu' else Advs


def _run(e, agent, lay, x, W):
    T = e.T
    e.T_cur = T
    e.obs_buf.zero_()
    e.obs_buf[:T, :, :, :W].copy_(to_dev(np.transpose(x['base'][:T], (0, 2, 1, 3))))
    e.fp_buf[:T].copy_(to_dev(np.transpose(x['fp'], (0, 2, 1, 3))))
    e.act_buf[:T].copy_(to_dev(np.transpose(x['acts'], (0, 2, 1)), torch.int32))
    e.done_buf[:T].copy_(to_dev(x['dones'][:T]))
    e.Rs[:T].copy_(to_dev(np.transpose(x['Rs'], (0, 2, 1))))
    e.Advs[:T].copy_(to_dev(np.transpose(_kernel_advs(agent, x['Advs']), (0, 2, 1))))
    e.set_states(nb(x['c0']), nb(x['h0']))
    e.backward()
    r = _result(e, lay)
    r['c'], r['h'] = _states(e, 1, T + 1)
    return r


def _oracle(agent, params, c, x, n_s, n_a, mask):
    """float64 oracle after one backward (gradients kept), with the round-off scales and the states it went through"""
    T, B, N = c['T'], c['B'], len(n_s)
    orc = HeteroIA2COracle(agent, n_s, n_a, mask, params=params, dtype=torch.float64, n_env=B)
    obs = [[x['base'][t][:, i, :n_s[i]] for i in range(N)] for t in range(T)]
    st = torch.tensor(np.concatenate([x['c0'], x['h0']], -1), dtype=torch.float64)
    orc.states_bw = st.clone()
    mode = RoundoffScale(orc.p)
    with mode:
        summ = orc.backward(obs, x['fp'].astype(np.float64), x['acts'], x['dones'][:T], x['Rs'], x['Advs'], 5e-4,
                            v_coef=HP['v_coef'], e_coef=HP['e_coef'], apply=False)
    cs, hs = [], []
    with torch.no_grad():
        cc, hh = st[..., :NH], st[..., NH:]
        for t in range(T):
            xt, pt = orc._prep(obs[t], x['fp'][t].astype(np.float64))
            cc, hh = orc._cell(xt, pt, torch.as_tensor(x['dones'][t], dtype=torch.float64), cc, hh)
            cs.append(cc.numpy()); hs.append(hh.numpy())
    ref = dict(g={n: orc.grads[n].numpy() for n in orc.names}, S={n: mode.S[n].numpy() for n in orc.names},
               K={n: mode.K[n].numpy() for n in orc.names}, summ=summ, c=np.stack(cs), h=np.stack(hs))
    return orc, ref


@pytest.mark.parametrize('name', GOLDEN)
@pytest.mark.parametrize('B', [7, 128, 256])                # 128, 256: tensor-core path
def test_hetero_ia2c_kernels_match_oracle(name, B):
    agent, lay, params, c, n_s, n_a = _setup(name, B)
    x = _inputs(c, n_s, n_a, seed=1)
    W, used, pad = max(n_s), _used(lay), _padding(lay)
    tc = B % 128 == 0
    tag = 'B=%d' % B
    e = _engine(lay, params, c, tc=tc)
    r = _run(e, agent, lay, x, W)                            # _result: synchronize + check_tc (tc_err == 0)
    orc, ref = _oracle(agent, params, c, x, n_s, n_a, lay.mask)
    ratios = _check(tag, r, ref, used)
    if tc:                                                   # per-entry error within 4x the FFMA kernels' + FLOOR
        e0 = _engine(lay, params, c, tc=False)
        r0 = _check(tag + ' ffma', _run(e0, agent, lay, x, W), ref, used)
        del e0
        bad = {n: (ratios[n], r0[n]) for n in ratios if ratios[n] > 4 * r0[n] + FLOOR}
        assert not bad, (tag, sorted(bad.items(), key=lambda t: -t[1][0])[:6])
    assert e.norm_out.numel() == (len(n_s) if agent != 'ma2c_cu' else 1)
    check_apply_twice(e, orc, lay, pad)
    e.check_tc()


@pytest.mark.parametrize('name', [p for p in GOLDEN if p.values[0].endswith('ma2c_cu')])
def test_hetero_cu_consensus_update_matches_oracle(name):
    from deeprl_network_b200.agents.engine import PolicyEngine
    agent, lay, params, c, n_s, n_a = _setup(name, 7)
    e = PolicyEngine(lay, c['B'], c['T'], dict(HP), flat_params=lay.pack(params))
    orc = HeteroIA2COracle(agent, n_s, n_a, lay.mask, params=params, dtype=torch.float64, n_env=c['B'])
    before = e.params.cpu().numpy().copy()
    e.grads.zero_()
    e.apply(1e-2)                      # zero gradients: clip + RMSProp leave the weights as they are, then the consensus
    torch.cuda.synchronize()
    with torch.no_grad():
        orc.consensus_update()
    flat = e.params.cpu().numpy()
    w = lay.unpack(flat)
    moved = set()
    for n in orc.names:
        np.testing.assert_allclose(w[n], orc.p[n].detach().numpy(), rtol=0, atol=1e-6, err_msg=n)
        if not np.array_equal(w[n], params[n]):
            moved.add(n)
    lstm = {n for n in orc.names if '/lstm_' in n}
    assert moved <= lstm and any(n.endswith('/wx') for n in moved)       # only the LSTM blocks are averaged
    for n in set(orc.names) - lstm:
        assert np.array_equal(w[n], params[n]), n
    assert np.array_equal(flat[_padding(lay)], before[_padding(lay)])
    iso = [i for i in range(len(n_s)) if not lay.nbr[i]]
    for i in iso:                      # an agent without neighbours averages over itself alone
        for k in ('wx', 'wh', 'b'):
            assert np.array_equal(w['cu/lstm_%da/%s' % (i, k)], params['cu/lstm_%da/%s' % (i, k)])
