"""CPU: heterogeneous IA2C / IA2C_FP / IA2C_CU (the reference's ``identical_agent == False`` path of LstmPolicy,
FPPolicy and ConsensusPolicy).

(1) HeteroLayout embeds the reference's tight tensors in the padded homogeneous model: names, shapes and creation
    order of tests/golden/hetero_*{ia2c,ia2c_fp,ma2c_cu}.npz, a one-to-one round trip, zeros everywhere else except
    the -1e30 bias of padded actions, and the observation gather the kernels get (IA2C / IA2C_FP: one source of the
    agent's own width; IA2C_CU: the agent's own row, padded to max(n_s)).
(2) The oracle (tests/hetero_ia2c_oracle.py) replays every fixture -- recorded from the UNMODIFIED reference classes
    on the TF shim with n_s = [5,7,4,6,5,3], n_a = [4,3,5,2,4,3], 3 updates of 8 steps, on the irregular graph and with
    the last ('iso') or first ('iso0') agent cut off: same initial weights from the same NumPy stream (exact), every
    pi / v / R within 1e-5, the sampled trained weights within 2e-5."""
import hashlib

import numpy as np
import pytest

from helpers import golden, load_cfg, random_params
from hetero_ia2c_oracle import HeteroIA2COracle
from test_hetero_parity import OracleHeteroAgent, replay, w1_error

AGENTS = ['ia2c', 'ia2c_fp', 'ma2c_cu']
GOLDEN = [pytest.param('hetero_%s%s' % (t, a), id='%s%s' % (t, a)) for t in ('', 'iso_', 'iso0_') for a in AGENTS]


def variant_of(name):
    """hetero_[iso_|iso0_]<agent> -> <agent>"""
    for t in ('hetero_iso0_', 'hetero_iso_', 'hetero_'):
        if name.startswith(t):
            return name[len(t):]


def full_obs(agent, nbr, ob, fp):
    """IA2C_FP: the environment appends the neighbours' last policies to every observation (make_golden_hetero_ia2c)"""
    if agent != 'ia2c_fp':
        return ob
    return [np.concatenate([ob[i]] + [np.asarray(fp[j], dtype=np.float64) for j in nbr[i]]) for i in range(len(ob))]


def replay_agent(g, agent, m):
    """Drive an agent with the reference API of `agent` (IA2C: forward(ob, done) / forward(ob, done, nactions, 'v');
    IA2C_CU: the MA2C signatures) through the recorded stream."""
    mask = g['mask']
    nbr = [list(np.where(mask[i] == 1)[0]) for i in range(len(mask))]
    if agent == 'ma2c_cu':
        return replay(g, lambda ob, d, fp: m.forward(ob, d, fp), lambda ob, d, fp, a: m.forward(ob, d, fp, a, 'v'),
                      m.add_transition, lambda R: m.backward(R, 0))
    nact = lambda a: [a[nbr[i]] for i in range(len(nbr))]
    return replay(g, lambda ob, d, fp: m.forward(full_obs(agent, nbr, ob, fp), d),
                  lambda ob, d, fp, a: m.forward(full_obs(agent, nbr, ob, fp), d, nact(a), 'v'),
                  lambda ob, fp, a, r, v, d: m.add_transition(full_obs(agent, nbr, ob, fp), nact(a), a, r, v, d),
                  lambda R: m.backward(R, 0))


@pytest.mark.parametrize('name', GOLDEN)
def test_hetero_ia2c_layout_embedding_round_trip(name):
    from deeprl_network_b200.layout import PI_PAD_BIAS, HeteroLayout
    agent, g = variant_of(name), golden(name)
    n_s, n_a, mask = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']], g['mask']
    lay = HeteroLayout(agent, n_s, n_a, mask)
    order = lay.creation_order()
    assert [n for n, _ in order] == [str(n) for n in g['names']]
    assert all(tuple(s) == tuple(g['w0shape/' + n]) for n, s in order)
    params = random_params(order, seed=3)
    flat = lay.pack(params)
    back = lay.unpack(flat)
    assert all(np.array_equal(back[n], params[n]) for n, _ in order)
    used = np.concatenate([lay._idx[n] for n, _ in order])
    assert len(used) == len(set(used.tolist())) == lay.n_real_param()
    rest = np.ones(lay.n_param, bool); rest[used] = False
    pad_bias = np.zeros(lay.n_param, bool); pad_bias[lay.pi_pad] = True
    assert np.all(flat[rest & ~pad_bias] == 0) and np.all(flat[pad_bias] == np.float32(PI_PAD_BIAS))
    assert len(lay.pi_pad) == sum(max(n_a) - a for a in n_a)
    m = lay.c_model()
    assert m.n_a == max(n_a) and lay.kx_pad <= 32 and lay.kp_pad <= 32
    for i in range(len(n_s)):
        ag = m.agent[i]
        assert ag.n_nbr == int(mask[i].sum()) and ag.x_nsrc == 1 and ag.x_src[0] == i
        assert ag.x_w == (max(n_s) if agent == 'ma2c_cu' else n_s[i])
    assert bool(m.per_agent_norm) == (agent != 'ma2c_cu')


def test_hetero_ia2c_fp_value_and_fingerprint_rows():
    """The one-hot of neighbour k's action a, and fingerprint entry a of neighbour k, sit at row k * max(n_a) + a of
    the padded value head / fcp; rows a >= n_a_j belong to no reference tensor."""
    from deeprl_network_b200.layout import NH, HeteroLayout
    g = golden('hetero_ia2c_fp')
    n_s, n_a, mask = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']], g['mask']
    lay = HeteroLayout('ia2c_fp', n_s, n_a, mask)
    na_max = max(n_a)
    for i in range(len(n_s)):
        nb = lay.nbr[i]
        o_fp, o_v = lay.agents_off[i]['o_w_fp'], lay.agents_off[i]['o_v_w']
        want_fp = [o_fp + (k * na_max + a) * NH + c for k, j in enumerate(nb) for a in range(n_a[j]) for c in range(NH)]
        assert lay._idx['lstm_%d/fcp/w' % i].tolist() == want_fp
        want_v = [o_v + r for r in range(NH)] + [o_v + NH + k * na_max + a for k, j in enumerate(nb) for a in range(n_a[j])]
        assert lay._idx['lstm_%d/v/w' % i].tolist() == want_v


class OracleHeteroIA2CAgent(OracleHeteroAgent):
    """The n-step returns and replay protocol of OracleHeteroAgent around HeteroIA2COracle.  With coop_gamma = -1
    every IA2C agent's OnPolicyBuffer computes the same returns as the multi-agent buffer; the per-agent loss, clip
    and optimizer live in the oracle."""

    def __init__(self, agent, g, mc):
        self.n_s, self.n_a = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']]
        np.random.seed(12)
        self.pol = HeteroIA2COracle(agent, self.n_s, self.n_a, g['mask'])
        self.mc, self.N = mc, len(self.n_s)
        self.buf = []


@pytest.mark.parametrize('name', GOLDEN)
def test_oracle_hetero_ia2c_follows_reference_on_tf_shim(name):
    agent, g = variant_of(name), golden(name)
    iso = {'hetero_iso_': [5], 'hetero_iso0': [0]}.get(name[:11], [])
    assert [i for i in range(len(g['mask'])) if g['mask'][i].sum() == 0] == iso
    ag = OracleHeteroIA2CAgent(agent, g, load_cfg('config_ma2c_nc_catchup.ini')['MODEL_CONFIG'])
    names = [str(n) for n in g['names']]
    assert names == ag.pol.names
    for n in names:
        w = np.ascontiguousarray(ag.pol.p[n].detach().numpy())
        assert w.shape == tuple(g['w0shape/' + n]), n
        assert hashlib.sha256(w.tobytes()).hexdigest() == str(g['w0sha/' + n]), n
    # the oracle takes IA2C_FP fingerprints as a separate array, so the MA2C-style protocol serves all three
    trace = replay(g, ag.policy, ag.value, ag.add, ag.backward)
    assert trace.shape == g['trace'].shape
    assert np.abs(trace - g['trace']).max() < 1e-5
    for n in names:
        assert w1_error(g, n, ag.pol.p[n].detach().numpy()) < 2e-5, n
