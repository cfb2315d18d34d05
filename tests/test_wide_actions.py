"""CPU: action counts 8 to 15 (the 16-wide head: n_a logits + the value slot).

Layouts of all six agents at n_a = 8, 11, 15 on the 8-agent chain, the 5x5 grid and the chain with one agent cut off
(names, shapes, creation order, pack / unpack with zero padding, the descriptor, the kernel family at B = 128); the
row width of sv_dlv and the head term of the workspace; the refusal of n_a = 16 by the layout and by the library; and
the float64 oracle replaying the reference's heterogeneous agents with 2 to 15 actions and its identical agents with 12
actions each (tests/golden/wide_*.npz, make_golden_wide_actions.py).  tests/test_gpu_wide_actions.py runs a subset of
these layouts on the device, chosen to reach every kernel family and instantiation.

Tensor-core eligibility does not depend on n_a except through the fingerprint encoder of NeurComm and ia2c_fp,
kp_pad = up4(n_a * neighbours) <= 32: the chain (2 neighbours) keeps the tensor cores up to n_a = 15 (kp = 32), the
4-neighbour grid up to n_a = 8 (kp = 32) and runs FFMA from n_a = 9 (kp = 36).  CommNet, DIAL, ia2c and ma2c_cu have
no fingerprint encoder, so n_a never moves them."""
import ctypes
import hashlib
from unittest import mock

import numpy as np
import pytest

import shape_cases
import test_shape_envelope
from helpers import golden, load_cfg
from shape_cases import Case
from test_hetero_ia2c_parity import OracleHeteroIA2CAgent
from test_hetero_parity import OracleHeteroAgent, replay, w1_error

FP_FAMILY = ('ma2c_nc', 'ia2c_fp')


def _case(variant, topo, n_a):
    kp = -(-n_a * (4 if topo == 'grid5' else 2) // 4) * 4
    return Case(variant, topo, 5, n_a, not (variant in FP_FAMILY and kp > 32), '16-wide head')


# the chain and the grid for all six agents; the cut chain for the agents that run an agent without neighbours
# (CommNet's mean over no neighbours is undefined)
WIDE = {}
for _na in (8, 11, 15):
    for _v in shape_cases.VARIANTS:
        for _topo in ('chain8', 'grid5', 'cut8'):
            if _topo == 'cut8' and _v == 'ma2c_ic3':
                continue
            WIDE['%s-%s-a%d' % (_v, _topo, _na)] = _case(_v, _topo, _na)
for _na in (9,):
    for _v in FP_FAMILY:
        WIDE['%s-grid5-a%d' % (_v, _na)] = _case(_v, 'grid5', _na)

# heterogeneous agents with 2 to 15 actions (wide_*, wide_iso_*: the last agent without neighbours) and identical agents
# with 12 actions each (wide_n12_*: the reference's identical_agent branch)
FIXTURES = ['wide_ma2c_nc', 'wide_ma2c_dial', 'wide_ia2c_fp', 'wide_iso_ia2c_fp', 'wide_n12_ma2c_nc']
HETERO_FIXTURES = [f for f in FIXTURES if not f.startswith('wide_n12_')]


def agent_of(name):
    """wide_[iso_|n12_]<agent> -> <agent>"""
    for t in ('wide_iso_', 'wide_n12_', 'wide_'):
        if name.startswith(t):
            return name[len(t):]


class OracleIdenticalAgent(OracleHeteroAgent):
    """OracleHeteroAgent's protocol for identical agents: one n_a for all, pi returned as one [B, N, n_a] array"""

    def __init__(self, agent, g, mc):
        from oracle import nets
        self.n_s, self.n_a = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']]
        np.random.seed(12)
        self.pol = nets.OraclePolicy(agent, self.n_s, self.n_a[0], g['mask'])
        self.mc, self.N = mc, len(self.n_s)
        self.buf = []

    def policy(self, ob, done, fp):
        return list(self.pol.forward(ob, done, fp, None, 'p')[0])


@pytest.mark.parametrize('cid', list(WIDE))
def test_wide_layout(cid):
    """test_shape_envelope's layout checks (formulas, packed operands, descriptor gather, pack / unpack with zero
    padding, kernel family at B = 128 / 256, never tensor cores on ragged env counts) on the wide cases"""
    with mock.patch.dict(shape_cases.CASES, {cid: WIDE[cid]}):
        test_shape_envelope.test_layout_of_case(cid)
    lay = shape_cases.layout_of(WIDE[cid])
    n_a, m = WIDE[cid].n_a, lay.c_model()
    assert m.n_a == n_a
    shapes = [s for n, _, s in lay.entries if n.split('/')[-2].startswith(('pi', 'v'))]
    want = [x for i in range(lay.N) for x in ((lay.n_h, n_a), (n_a,), (lay.n_h + n_a * len(lay.nbr[i]), 1), (1,))]
    assert sorted(shapes) == sorted(want)


def test_kernel_family_at_the_fingerprint_boundary():
    """The cases the tensor-core predicate turns on, stated on the layouts (B = 128)."""
    from deeprl_network_b200.agents.engine import tc_eligible
    lay = lambda v, topo, n_a: shape_cases.layout_of(_case(v, topo, n_a))
    for v in FP_FAMILY:
        assert lay(v, 'chain8', 15).kp_pad == 32 and tc_eligible(lay(v, 'chain8', 15), 128)
        assert lay(v, 'grid5', 8).kp_pad == 32 and tc_eligible(lay(v, 'grid5', 8), 128)
        assert lay(v, 'grid5', 9).kp_pad == 36 and not tc_eligible(lay(v, 'grid5', 9), 128)
    for v in ('ma2c_ic3', 'ma2c_dial', 'ia2c', 'ma2c_cu'):
        for n_a in (8, 15):
            assert lay(v, 'grid5', n_a).kp_pad == 0 and tc_eligible(lay(v, 'grid5', n_a), 128)


def test_descriptor_size_and_head_width():
    from deeprl_network_b200 import _lib as L
    lib = L.lib()
    assert L.MAX_NA == 16
    assert ctypes.sizeof(L.Model) == lib.nmarl_sizeof_model() == 48 + 128 * 192
    assert lib.nmarl_version() >= 104
    assert [L.head_width(n) for n in range(1, 16)] == [8] * 7 + [16] * 8


def test_workspace_head_term():
    """nmarl_ws_floats covers the head weight-gradient workspace, head_splits x N x head_ws(HW) floats with
    head_ws = 64 HW + HW + 4 HW: 552 for n_a <= 7, 1 104 for n_a 8..15.  On a 128-agent chain at n_h = 16 and 2^19 rows
    (head_splits = 512) that term is larger than the weight-gradient GEMMs' workspace, so it decides the total:
    512 x 128 x 552 = 36 175 872 floats for n_a <= 7 (what the library returned before the 16-wide head existed) and
    twice that from n_a = 8 on."""
    from deeprl_network_b200 import _lib as L
    from deeprl_network_b200.layout import ModelLayout
    from oracle.cacc import chain_masks
    mask = chain_masks(128)[0]

    def ws(n_a):
        lay = ModelLayout('ia2c', [5 * (1 + int(k)) for k in mask.sum(1)], n_a, mask, n_h=16, n_fc=16)
        return int(L.lib().nmarl_ws_floats(ctypes.byref(lay.c_model()), 4096, 128))
    assert ws(1) == ws(4) == ws(7) == 512 * 128 * 552 == 36175872
    assert ws(8) == ws(11) == ws(15) == 512 * 128 * 1104


def test_n_a_16_is_refused():
    from deeprl_network_b200 import _lib as L
    from deeprl_network_b200.layout import HeteroLayout, ModelLayout
    from oracle.cacc import chain_masks
    mask = chain_masks(8)[0]
    with pytest.raises(ValueError, match='15'):
        ModelLayout('ma2c_nc', [5] * 8, 16, mask)
    with pytest.raises(ValueError, match='15'):
        HeteroLayout('ma2c_dial', [5] * 8, [3, 16, 4, 4, 4, 4, 4, 4], mask)
    m = ModelLayout('ma2c_nc', [5] * 8, 15, mask).c_model()
    m.n_a = 16
    lib = L.lib()
    assert lib.nmarl_policy_step_p(ctypes.byref(m), ctypes.byref(L.FwdArgs()), None) != 0
    assert b'n_a 16 out of range (max 15)' in lib.nmarl_last_error()


@pytest.mark.parametrize('name', HETERO_FIXTURES)
def test_wide_fixture_layout(name):
    from deeprl_network_b200.layout import PI_PAD_BIAS, HeteroLayout
    from helpers import random_params
    g = golden(name)
    agent = agent_of(name)
    n_s, n_a, mask = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']], g['mask']
    assert max(n_a) == 15 and min(n_a) < 8
    lay = HeteroLayout(agent, n_s, n_a, mask)
    order = lay.creation_order()
    assert [n for n, _ in order] == [str(n) for n in g['names']]
    assert all(tuple(s) == tuple(g['w0shape/' + n]) for n, s in order)
    params = random_params(order, seed=3)
    flat = lay.pack(params)
    assert all(np.array_equal(lay.unpack(flat)[n], params[n]) for n, _ in order)
    assert np.all(flat[lay.pi_pad] == np.float32(PI_PAD_BIAS)) and len(lay.pi_pad) == sum(15 - a for a in n_a)


@pytest.mark.parametrize('name', FIXTURES)
def test_oracle_follows_reference_with_wide_heads(name):
    """Same initial weights from the same NumPy stream (exact), every pi / v / R within 1e-5, the trained weights'
    sample within 2e-5 -- heterogeneous agents, and identical ones with 12 actions each."""
    g = golden(name)
    agent = agent_of(name)
    iso = [5] if name.startswith('wide_iso_') else []
    assert [i for i in range(len(g['mask'])) if g['mask'][i].sum() == 0] == iso
    same = name.startswith('wide_n12_')
    assert (len(set(g['n_a_ls'].tolist())) == 1) == same and max(g['n_a_ls']) >= 12
    mc = load_cfg('config_ma2c_nc_catchup.ini')['MODEL_CONFIG']
    cls = OracleIdenticalAgent if same else (OracleHeteroIA2CAgent if agent == 'ia2c_fp' else OracleHeteroAgent)
    ag = cls(agent, g, mc)
    names = [str(n) for n in g['names']]
    assert names == ag.pol.names
    for n in names:
        w = np.ascontiguousarray(ag.pol.p[n].detach().numpy())
        assert w.shape == tuple(g['w0shape/' + n]), n
        assert hashlib.sha256(w.tobytes()).hexdigest() == str(g['w0sha/' + n]), n
    trace = replay(g, ag.policy, ag.value, ag.add, ag.backward)
    assert trace.shape == g['trace'].shape
    assert np.abs(trace - g['trace']).max() < 1e-5
    for n in names:
        assert w1_error(g, n, ag.pol.p[n].detach().numpy()) < 2e-5, n
