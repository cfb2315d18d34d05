"""CPU: LSTM widths num_lstm = 16 and 32.

(1) Host layouts: names, shapes and creation order equal the reference's at that width (oracle/nets.param_shapes, and
    tests/hetero_ia2c_oracle.param_shapes for the heterogeneous IA2C family), pack / unpack round-trip, the descriptor
    carries the width through s_dim, and unsupported widths -- or ia2c / ia2c_fp with num_fc != num_lstm -- are refused.
(2) The float64 oracle replays the fixtures recorded from the UNMODIFIED reference on the TF shim at these widths
    (tests/golden/make_golden_hidden.py): tfnet_h{16,32}_<agent> (env + Trainer + agent class, as
    tests/test_tfnet_parity.py) and hetero_h32_{ma2c_nc,ia2c_fp} (heterogeneous agents, the last one without
    neighbours, as tests/test_hetero_parity.py).  Same initial weights from the same NumPy stream (exact), every
    pi / v / R within 1e-5, the sampled trained weights within 2e-5.
"""
import ctypes
import hashlib

import numpy as np
import pytest

from helpers import golden, load_cfg, random_params
from oracle import nets
from oracle.cacc import OracleCACC, chain_masks
from oracle.trainer import Counter, OracleAgent, OracleTrainer

import hetero_ia2c_oracle
from test_hetero_ia2c_parity import OracleHeteroIA2CAgent
from test_hetero_parity import OracleHeteroAgent, replay, w1_error
from test_tfnet_parity import Rec

VARIANTS = ['ia2c', 'ia2c_fp', 'ma2c_cu', 'ma2c_nc', 'ma2c_ic3', 'ma2c_dial']
N_A = 4


def _homo(variant, n_h, n_fc=None):
    from deeprl_network_b200.layout import ModelLayout
    mask, _ = chain_masks(8)
    nm = [int(mask[i].sum()) for i in range(8)]
    n_s_ls = {'ia2c': [5 * (1 + k) for k in nm], 'ia2c_fp': [5 * (1 + k) + N_A * k for k in nm]}.get(variant, [5] * 8)
    lay = ModelLayout(variant, n_s_ls, N_A, mask, n_h=n_h, n_fc=n_h if n_fc is None else n_fc, obs_mode='gather')
    return lay, n_s_ls, mask


def _shapes(want):
    return [(n, tuple(s)) for n, s in (want.items() if isinstance(want, dict) else want)]


@pytest.mark.parametrize('n_h', [16, 32])
@pytest.mark.parametrize('variant', VARIANTS)
def test_homogeneous_layout_follows_reference(variant, n_h):
    lay, n_s_ls, mask = _homo(variant, n_h)
    want = _shapes(nets.param_shapes(variant, n_s_ls, N_A, mask, n_h=n_h, n_fc=n_h))
    assert [(n, tuple(s)) for n, s in lay.creation_order()] == want
    assert lay.n_h == n_h
    assert lay.s_dim == (3 * n_h if variant in ('ma2c_nc', 'ia2c_fp') else n_h)
    assert lay.km_pad == {'ia2c': 0, 'ma2c_cu': 0, 'ma2c_ic3': n_h}.get(variant, 2 * n_h)     # chain: <= 2 neighbours
    params = random_params(lay.creation_order(), seed=1)
    back = lay.unpack(lay.pack(params))
    assert set(back) == set(params) and all(np.array_equal(back[k], params[k]) for k in params)
    m = lay.c_model()
    assert m.s_dim == lay.s_dim and (m.kx_pad, m.kp_pad, m.km_pad) == (lay.kx_pad, lay.kp_pad, lay.km_pad)
    assert m.n_param == lay.n_param and m.n_param < _homo(variant, 64)[0].n_param
    for i in range(8):
        ag = m.agent[i]
        assert ag.o_b - ag.o_wxh == (lay.s_dim + n_h) * 4 * n_h            # [wx; wh] is one [s_dim + n_h, 4 n_h] block
        assert ag.t_wxh + 4 * n_h * (lay.s_dim + n_h) <= m.n_wt


def test_reference_names_at_width_32():
    lay, _, _ = _homo('ma2c_nc', 32)
    assert lay.by_name['nc/lstm_comm_1/wx_hid'][1] == (96, 128)
    assert lay.by_name['nc/lstm_comm_1/wh_hid'][1] == (32, 128)
    assert lay.by_name['nc/lstm_comm_1/w_msg'][1] == (64, 32)
    assert lay.by_name['nc/v_1/w'][1] == (32 + 2 * N_A, 1)
    lay, _, _ = _homo('ma2c_dial', 16)
    assert lay.by_name['dial/mfc_0/w'][1] == (16, 16)


HETERO = ['hetero_ma2c_nc', 'hetero_iso_ma2c_nc', 'hetero_iso_ma2c_dial', 'hetero_ma2c_ic3',
          'hetero_ia2c', 'hetero_iso_ia2c_fp', 'hetero_ma2c_cu']


@pytest.mark.parametrize('n_h', [16, 32])
@pytest.mark.parametrize('name', HETERO)
def test_heterogeneous_layout_follows_reference(name, n_h):
    from deeprl_network_b200.layout import HeteroLayout
    variant = name.split('_', 2)[-1] if name.startswith('hetero_iso_') else name[len('hetero_'):]
    g = golden(name)
    n_s, n_a, mask = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']], g['mask']
    lay = HeteroLayout(variant, n_s, n_a, mask, n_h=n_h, n_fc=n_h)
    if variant in ('ia2c', 'ia2c_fp', 'ma2c_cu'):
        want = hetero_ia2c_oracle.param_shapes(variant, n_s, n_a, mask, n_h=n_h, n_fc=n_h)
    else:
        want = nets.param_shapes(variant, n_s, n_a, mask, n_h=n_h, n_fc=n_h)
    assert [(n, tuple(s)) for n, s in lay.creation_order()] == _shapes(want)
    params = random_params(lay.creation_order(), seed=2)
    flat = lay.pack(params)
    back = lay.unpack(flat)
    assert all(np.array_equal(back[k], params[k]) for k in params)
    m = lay.c_model()
    assert m.s_dim == (3 * n_h if lay.vid == 1 else n_h)


@pytest.mark.parametrize('variant', ['ma2c_nc', 'ma2c_ic3', 'ma2c_dial', 'ma2c_cu'])
def test_num_fc_is_ignored_where_the_reference_ignores_it(variant):
    a, _, _ = _homo(variant, 32, n_fc=32)
    b, _, _ = _homo(variant, 32, n_fc=128)
    assert a.creation_order() == b.creation_order() and a.n_param == b.n_param


def test_unsupported_widths_fail_loudly():
    for n_h in (48, 128, 8):
        with pytest.raises(ValueError, match='num_lstm = %d' % n_h):
            _homo('ma2c_nc', n_h)
    for variant in ('ia2c', 'ia2c_fp'):
        with pytest.raises(ValueError, match='num_fc = 16, num_lstm = 32'):
            _homo(variant, 32, n_fc=16)


def test_descriptor_size_is_unchanged():
    from deeprl_network_b200 import _lib as L
    assert ctypes.sizeof(L.Model) == 48 + 128 * 192                # the width travels in s_dim


# ---- fixtures recorded from the reference at widths 16 / 32 --------------------------------------------------------
TFNET_H = ['tfnet_h%d_%s' % (h, a) for h in (16, 32)
           for a in ('ma2c_nc', 'ia2c', 'ia2c_fp', 'ma2c_ic3', 'ma2c_dial', 'ma2c_cu')]


def width_cfg(ini, n_h):
    """the shipped config with MODEL_CONFIG num_lstm = num_fc = n_h, as the fixture was recorded"""
    cp = load_cfg(ini)
    cp['MODEL_CONFIG']['num_lstm'] = str(n_h)
    cp['MODEL_CONFIG']['num_fc'] = str(n_h)
    return cp


@pytest.mark.parametrize('name', TFNET_H)
def test_oracle_follows_reference_at_narrow_width(name):
    g = golden(name)
    n_h = int(g['n_h'])
    cp = width_cfg(str(g['ini']), n_h)
    env = OracleCACC(cp['ENV_CONFIG'])
    agent = OracleAgent(env.agent, env.n_s_ls, env.n_a_ls, env.neighbor_mask, env.distance_mask, env.coop_gamma,
                        10 ** 6, cp['MODEL_CONFIG'], seed=12)
    names = [str(n) for n in g['names']]
    assert sorted(names) == sorted(agent.policy.names)
    for n in names:                                                       # creation order + ortho init reproduce w0
        w = np.ascontiguousarray(agent.policy.p[n].detach().numpy())
        assert w.shape == tuple(g['w0shape/' + n]), n
        assert hashlib.sha256(w.tobytes()).hexdigest() == str(g['w0sha/' + n]), n
    w0 = {n: agent.policy.p[n].detach().numpy().copy() for n in names}
    rec = Rec(agent)
    counter = Counter(int(g['total_step']), 10 ** 9, 10 ** 9)
    OracleTrainer(env, rec, counter).run()
    assert counter.cur_step == int(g['cur_step']) and env.seed == int(g['seed_after'])
    trace = np.concatenate(rec.log)
    assert trace.shape == g['trace'].shape
    assert np.abs(trace - g['trace']).max() < 1e-5
    for n in names:
        assert w1_error(g, n, agent.policy.p[n].detach().numpy()) < 2e-5, n
    assert max(w1_error(g, n, w0[n]) for n in names) > 1e-3               # training moved the weights


class WidthHeteroAgent(OracleHeteroAgent):
    """OracleHeteroAgent at the fixture's width"""

    def __init__(self, agent, g, mc):
        super().__init__(agent, g, mc)
        np.random.seed(12)
        self.pol = nets.OraclePolicy(agent, self.n_s, self.n_a, g['mask'], n_h=int(g['n_h']), n_fc=int(g['n_h']))


class WidthHeteroIA2CAgent(OracleHeteroIA2CAgent):
    """OracleHeteroIA2CAgent at the fixture's width"""

    def __init__(self, agent, g, mc):
        super().__init__(agent, g, mc)
        np.random.seed(12)
        self.pol = hetero_ia2c_oracle.HeteroIA2COracle(agent, self.n_s, self.n_a, g['mask'], n_h=int(g['n_h']),
                                                       n_fc=int(g['n_h']))


@pytest.mark.parametrize('name', ['hetero_h32_ma2c_nc', 'hetero_h32_ia2c_fp'])
def test_oracle_hetero_follows_reference_at_width_32(name):
    from deeprl_network_b200.layout import HeteroLayout
    g = golden(name)
    agent = name[len('hetero_h32_'):]
    assert int(g['n_h']) == 32
    assert [i for i in range(len(g['mask'])) if g['mask'][i].sum() == 0] == [5]      # the last agent is cut off
    mc = width_cfg('config_ma2c_nc_catchup.ini', 32)['MODEL_CONFIG']
    ag = (WidthHeteroIA2CAgent if agent == 'ia2c_fp' else WidthHeteroAgent)(agent, g, mc)
    names = [str(n) for n in g['names']]
    assert names == ag.pol.names
    lay = HeteroLayout(agent, [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']], g['mask'], n_h=32, n_fc=32)
    assert [(n, tuple(s)) for n, s in lay.creation_order()] == [(n, tuple(g['w0shape/' + n])) for n in names]
    for n in names:
        w = np.ascontiguousarray(ag.pol.p[n].detach().numpy())
        assert w.shape == tuple(g['w0shape/' + n]), n
        assert hashlib.sha256(w.tobytes()).hexdigest() == str(g['w0sha/' + n]), n
    trace = replay(g, ag.policy, ag.value, ag.add, ag.backward)
    assert trace.shape == g['trace'].shape
    assert np.abs(trace - g['trace']).max() < 1e-5
    for n in names:
        assert w1_error(g, n, ag.pol.p[n].detach().numpy()) < 2e-5, n
