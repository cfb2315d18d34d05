"""CPU: heterogeneous agents (SURVEY 8 f4, policy half) -- the oracle's restatement of lstm_comm_hetero /
lstm_ic3_hetero / lstm_dial_hetero + per-agent heads (agents/utils.py:220-341, 420-512, 602-702; agents/policies.py:
289, 453, 502; agents/models.py:89-97, 229-235) against the UNMODIFIED reference classes run on the TF shim
(tests/golden/make_golden.py::hetero_case -> tests/golden/hetero_*.npz): 6 agents on an irregular graph with
n_s = [5,7,4,6,5,3], n_a = [4,3,5,2,4,3], a scripted observation / reward / uniform stream, 3 updates of 8 steps.
The hetero_iso_* / hetero_iso0_* fixtures cut the last / the first agent off (NeurComm and DIAL: such an agent has no
message or fingerprint encoder).  Same initial weights from the same NumPy stream (exact), same sampled actions, every
pi / v / R within 1e-5, weights after the three updates within 2e-5 (the hetero_iso* fixtures keep a fixed sample of 256
entries of every larger tensor, see w1_error)."""
import hashlib

import numpy as np
import pytest

from helpers import golden, load_cfg
from oracle import nets

AGENTS = ['ma2c_nc', 'ma2c_ic3', 'ma2c_dial']
# (fixture, test id): the irregular graph, then the same agents with the last ('iso') or the first ('iso0') agent
# without neighbours
GOLDEN = ([pytest.param('hetero_' + a, id=a) for a in AGENTS] +
          [pytest.param('hetero_%s_%s' % (t, a), id='%s-%s' % (t, a)) for t in ('iso', 'iso0') for a in ('ma2c_nc', 'ma2c_dial')])


def w1_error(g, n, w):
    """max |w - trained reference weights| over the entries the fixture keeps: all of them, or (hetero_iso*) the
    fixed sample of flat indices 'w1idx/<name>' (tests/golden/make_golden.py::W1_SAMPLE)"""
    if 'w1idx/' + n in g.files:
        w = np.ascontiguousarray(w).ravel()[g['w1idx/' + n]]
    return np.abs(w - g['w1/' + n]).max()


def variant_of(name):
    """hetero_[iso_|iso0_]<agent> -> <agent>"""
    return name[name.index('ma2c_'):]


def replay(g, policy_fwd, value_fwd, add, backward):
    """Drive `policy_fwd(ob, done, fp) -> list of pi_i`, `value_fwd(ob, done, fp, act) -> v[N]`, `add(...)`,
    `backward(R)` with the recorded stream; returns the trace in the recording's order."""
    n_s, n_a = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']]
    N, T = len(n_s), int(g['n_step'])
    obs = g['obs'].reshape(-1, sum(n_s))
    cuts = np.cumsum([0] + n_s)
    uni, rew = g['uniforms'], g['rewards']
    log, k_obs, k_uni, k_rew = [], 0, 0, 0
    fp = [np.ones(n) / n for n in n_a]
    done = True

    def decide(ob, done, fp):
        nonlocal k_uni
        pi = [np.asarray(p, dtype=np.float64).ravel() for p in policy_fwd(ob, done, fp)]
        log.append(np.concatenate(pi))
        act = []
        for i in range(N):
            cdf = np.cumsum(pi[i]); cdf = cdf / cdf[-1]
            act.append(int(np.searchsorted(cdf, uni[k_uni][i], side='right')))
        k_uni += 1
        return pi, np.array(act)
    for _ in range(int(g['updates'])):
        for t in range(T):
            ob = [obs[k_obs][cuts[i]:cuts[i + 1]] for i in range(N)]; k_obs += 1
            pi, act = decide(ob, done, fp)
            v = np.asarray(value_fwd(ob, done, fp, act), dtype=np.float64).ravel()
            log.append(v)
            add(ob, fp, act, float(rew[k_rew]), v, False); k_rew += 1
            fp = [np.asarray(p, dtype=np.float32) for p in pi]
            done = False
        ob = [obs[k_obs][cuts[i]:cuts[i + 1]] for i in range(N)]; k_obs += 1
        pi, act = decide(ob, done, fp)
        R = np.asarray(value_fwd(ob, done, fp, act), dtype=np.float64).ravel()
        log.append(R)
        backward(R)
    return np.concatenate(log)


class OracleHeteroAgent:
    """MA2C_* agent protocol (add_transition / backward with the n-step returns) around OraclePolicy."""

    def __init__(self, agent, g, mc):
        self.n_s, self.n_a = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']]
        np.random.seed(12)
        self.pol = nets.OraclePolicy(agent, self.n_s, self.n_a, g['mask'])
        self.mc, self.N = mc, len(self.n_s)
        self.buf = []

    def policy(self, ob, done, fp):
        return [p[0] for p in self.pol.forward(ob, done, fp, None, 'p')]

    def value(self, ob, done, fp, act):
        return self.pol.forward(ob, done, fp, act[None], 'v')[0]

    def add(self, ob, fp, act, r, v, done):
        self.buf.append((ob, fp, act, r / self.mc.getfloat('reward_norm'), v, done))

    def backward(self, R_end):
        from oracle.buffers import nstep_returns
        T = len(self.buf)
        r = np.array([[b[3]] * self.N for b in self.buf]); v = np.array([b[4] for b in self.buf])
        Rs, Advs = nstep_returns(r, v, [b[5] for b in self.buf], R_end, self.mc.getfloat('gamma'))
        dones = np.array([[float(self._prev_done if t == 0 else self.buf[t - 1][5])] for t in range(T)])
        pad = lambda fp: np.stack([np.pad(np.asarray(q, dtype=np.float64), (0, max(self.n_a) - len(q))) for q in fp])[None]
        self.pol.backward([[np.asarray(o)[None] for o in b[0]] for b in self.buf], np.stack([pad(b[1]) for b in self.buf]),
                          np.array([b[2][None] for b in self.buf]), dones, Rs.T[:, None, :], Advs.T[:, None, :],
                          self.mc.getfloat('lr_init'), v_coef=self.mc.getfloat('value_coef'), e_coef=self.mc.getfloat('entropy_coef'),
                          max_grad_norm=self.mc.getfloat('max_grad_norm'), alpha=self.mc.getfloat('rmsp_alpha'),
                          epsilon=self.mc.getfloat('rmsp_epsilon'))
        self._prev_done = self.buf[-1][5]
        self.buf = []
    _prev_done = False         # quirk Q6: the reference buffer starts with done=False (agents/utils.py:731-738)


@pytest.mark.parametrize('name', GOLDEN)
def test_oracle_hetero_follows_reference_on_tf_shim(name):
    g = golden(name)
    iso = {'hetero_iso_': [5], 'hetero_iso0': [0]}.get(name[:11], [])
    assert [i for i in range(len(g['mask'])) if g['mask'][i].sum() == 0] == iso   # the agents the fixture cuts off
    mc = load_cfg('config_ma2c_nc_catchup.ini')['MODEL_CONFIG']
    ag = OracleHeteroAgent(variant_of(name), g, mc)
    names = [str(n) for n in g['names']]
    assert names == ag.pol.names                                          # creation order, one for one
    for n in names:
        w = np.ascontiguousarray(ag.pol.p[n].detach().numpy())
        assert w.shape == tuple(g['w0shape/' + n]), n
        assert hashlib.sha256(w.tobytes()).hexdigest() == str(g['w0sha/' + n]), n
    trace = replay(g, ag.policy, ag.value, ag.add, ag.backward)
    assert trace.shape == g['trace'].shape
    assert np.abs(trace - g['trace']).max() < 1e-5
    for n in names:
        assert w1_error(g, n, ag.pol.p[n].detach().numpy()) < 2e-5, n
