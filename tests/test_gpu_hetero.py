"""GPU: heterogeneous agents (SURVEY 8 f4, policy half) on the CUDA path.
(1) The drop-in agent classes (host lists in, NumPy out, B = 1) replay the scripted stream of
    tests/golden/hetero_*.npz -- recorded from the UNMODIFIED reference MA2C_NC / MA2C_IC3 / MA2C_DIAL classes with
    n_s = [5,7,4,6,5,3], n_a = [4,3,5,2,4,3] on the TF shim -- and must reproduce every pi / v / R within 1e-5 and the
    weights after three updates within 2e-5, starting from the same NumPy-stream initial weights (exact).
    The hetero_iso_* / hetero_iso0_* fixtures cut the last / the first agent off: it has no message or fingerprint
    encoder, so its b_fp / b_msg (and for NeurComm wx_hid rows 64..191) are padding of the embedding and must stay
    exactly 0; a DIAL agent without neighbours also adds no one-hot of its own action (lstm_dial_hetero).
(2) The batched kernels (FFMA and tensor-core paths) against the batched oracle: pi / v / state 1e-5, gradients
    2e-5 x scale against float64 autograd, and the zero-padding of the embedding receives exactly zero gradient;
    then two optimizer steps: norm_out equals the oracle's global norm and the padding stays exactly 0."""
import hashlib

import numpy as np
import pytest
import torch

from gpu_common import HP, bn, check_apply_twice, nb, to_dev
from helpers import golden, load_cfg, random_params
from oracle import nets
from test_hetero_parity import GOLDEN, replay, variant_of, w1_error

pytestmark = pytest.mark.gpu


def _padding(lay):
    """flat-buffer floats that belong to no reference tensor and are not a padded action's bias: exactly 0 for good"""
    pad = np.ones(lay.n_param, bool)
    for n in lay._idx:
        pad[lay._idx[n]] = False
    pad[lay.pi_pad] = False
    return pad


@pytest.mark.parametrize('name', GOLDEN)
def test_drop_in_agent_follows_reference_hetero_golden(name):
    from deeprl_network_b200.agents.models import MA2C_DIAL, MA2C_IC3, MA2C_NC
    agent = variant_of(name)
    g = golden(name)
    mc = load_cfg('config_ma2c_nc_catchup.ini')['MODEL_CONFIG']
    mc['batch_size'] = str(int(g['n_step']))
    n_s, n_a = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']]
    cls = {'ma2c_nc': MA2C_NC, 'ma2c_ic3': MA2C_IC3, 'ma2c_dial': MA2C_DIAL}[agent]
    np.random.seed(12)
    m = cls(n_s, n_a, g['mask'], np.zeros_like(g['mask']), -1.0, 10 ** 6, mc, seed=12)
    assert not m.identical_agent
    w0 = m.get_weights()
    names = [str(n) for n in g['names']]
    assert names == [n for n, _ in m.layout.creation_order()]
    for n in names:
        assert hashlib.sha256(np.ascontiguousarray(w0[n]).tobytes()).hexdigest() == str(g['w0sha/' + n]), n
    m.reset()
    trace = replay(g, lambda ob, d, fp: m.forward(ob, d, fp), lambda ob, d, fp, a: m.forward(ob, d, fp, a, 'v'),
                   m.add_transition, lambda R: m.backward(R, 0))
    assert trace.shape == g['trace'].shape
    assert np.abs(trace - g['trace']).max() < 1e-5
    w1 = m.get_weights()
    for n in names:
        assert w1_error(g, n, w1[n]) < 2e-5, n
    flat = m.engine.params.cpu().numpy()
    assert np.all(flat[m.layout.pi_pad] == np.float32(-1e30))           # padded actions never moved
    # the rest of the padding -- an isolated agent's b_fp / b_msg and unused wx_hid rows included -- never moved either
    assert np.all(flat[_padding(m.layout)] == 0)


def _pair(name, B, T):
    from deeprl_network_b200.agents.engine import PolicyEngine
    from deeprl_network_b200.layout import HeteroLayout
    agent = variant_of(name)
    g = golden(name)
    n_s, n_a, mask = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']], g['mask']
    lay = HeteroLayout(agent, n_s, n_a, mask)
    params = random_params(lay.creation_order(), seed=2, scale=0.3)
    eng = PolicyEngine(lay, B, T, dict(HP), flat_params=lay.pack(params))
    orc = nets.OraclePolicy(agent, n_s, n_a, mask, params=params, dtype=torch.float64, n_env=B)
    return eng, orc, lay, n_s, n_a


def _inputs(rs, shape, n_s, n_a):
    """padded observations [.., N, n_s_max] and fingerprints [.., N, n_a_max] with zeros beyond each agent's width"""
    N = len(n_s)
    ob = rs.randn(*shape, N, max(n_s)).astype(np.float32)
    fp = np.zeros((*shape, N, max(n_a)), dtype=np.float32)
    for i in range(N):
        ob[..., i, n_s[i]:] = 0
        fp[..., i, :n_a[i]] = rs.dirichlet(np.ones(n_a[i]), size=shape)
    return ob, fp


@pytest.mark.parametrize('name', GOLDEN)
@pytest.mark.parametrize('B', [7, 128])                     # 128: tensor-core path
def test_hetero_kernels_match_oracle(name, B):
    T = 4
    eng, orc, lay, n_s, n_a = _pair(name, B, T)
    assert eng.use_tc == (B % 128 == 0)
    N = len(n_s)
    rs = np.random.RandomState(1)
    ob, fp = _inputs(rs, (T, B), n_s, n_a)
    acts = np.stack([rs.randint(0, n_a[i], size=(T, B)) for i in range(N)], axis=-1)
    dones = np.zeros((T, B), dtype=np.float32); dones[0, ::2] = 1
    Rs = rs.randn(T, B, N).astype(np.float32); Advs = rs.randn(T, B, N).astype(np.float32)
    c0 = (rs.randn(B, N, 64) * .5).astype(np.float32); h0 = (rs.rand(B, N, 64) - .5).astype(np.float32)
    # ---- forward p / v ------------------------------------------------------------------------------------
    eng.set_states(nb(c0), nb(h0))
    orc.states_fw = torch.tensor(np.concatenate([c0, h0], -1), dtype=torch.float64)
    obs_d = torch.zeros(N, B, lay.obs_stride, device='cuda'); obs_d[:, :, :max(n_s)] = nb(ob[0])
    pi_d = torch.zeros(N, B, max(n_a), device='cuda'); v_d = torch.zeros(N, B, device='cuda')
    eng.step_p(obs_d, nb(fp[0]), to_dev(dones[0]), pi_d)
    pi_o = orc.forward([ob[0][:, i, :n_s[i]] for i in range(N)], dones[0], fp[0].astype(np.float64), None, 'p')
    pk = bn(pi_d)
    for i in range(N):
        np.testing.assert_allclose(pk[:, i, :n_a[i]], pi_o[i], rtol=0, atol=1e-5)
        assert np.all(pk[:, i, n_a[i]:] == 0)                # a padded action has probability exactly 0
    np.testing.assert_allclose(bn(eng.get_states_fw()), orc.states_fw.numpy(), rtol=0, atol=1e-5)
    eng.step_v(obs_d, nb(fp[0]), to_dev(dones[0]), nb(acts[0]).int(), v_d)
    v_o = orc.forward([ob[0][:, i, :n_s[i]] for i in range(N)], dones[0], fp[0].astype(np.float64), acts[0], 'v')
    np.testing.assert_allclose(bn(v_d), v_o, rtol=0, atol=1e-5)
    eng.check_tc()
    # ---- backward (quirk Q7: the kernels get the advantages summed over agents, see engine.compute_returns) ----
    eng.T_cur = T
    eng.obs_buf[:T].zero_(); eng.obs_buf[:T, :, :, :max(n_s)].copy_(to_dev(np.transpose(ob, (0, 2, 1, 3))))
    eng.fp_buf[:T].copy_(to_dev(np.transpose(fp, (0, 2, 1, 3))))
    eng.act_buf[:T].copy_(to_dev(np.transpose(acts, (0, 2, 1)), torch.int32))
    eng.done_buf[:T].copy_(to_dev(dones))
    eng.Rs[:T].copy_(to_dev(np.transpose(Rs, (0, 2, 1))))
    eng.Advs[:T].copy_(to_dev(np.transpose(np.repeat(Advs.sum(-1, keepdims=True), N, -1), (0, 2, 1))))
    eng.set_states(nb(c0), nb(h0))
    st = torch.tensor(np.concatenate([c0, h0], -1), dtype=torch.float64)
    orc.states_bw, orc.states_fw = st.clone(), st.clone()
    orc.backward([[ob[t][:, i, :n_s[i]] for i in range(N)] for t in range(T)], fp.astype(np.float64), acts, dones, Rs, Advs, 5e-4,
                 v_coef=HP['v_coef'], e_coef=HP['e_coef'], apply=False)
    eng.backward()
    torch.cuda.synchronize()
    eng.check_tc()
    flat = eng.grads.cpu().numpy()
    gk = lay.unpack(flat)
    for n in orc.names:
        ref = orc.grads[n].numpy()
        err, scale = np.abs(gk[n] - ref).max(), max(1e-3, np.abs(ref).max())
        assert err <= 2e-5 * scale + 1e-7, (n, err, scale)
    used = np.zeros(lay.n_param, bool)
    for n in orc.names:
        used[lay._idx[n]] = True
    assert np.all(flat[~used] == 0)                           # the zero-padding of the embedding gets zero gradient
    check_apply_twice(eng, orc, lay, _padding(lay))
