"""Host: the case table of tests/test_gpu_narrow_widths.py, the shared-memory boundary at each LSTM width, and the
float64 oracle against the reference at num_lstm = 16 with 12 actions per agent.

* Every case's layout is in the regime the case is named after (check_regime), and the table as a whole reaches every
  FP32-FFMA kernel instantiation the dispatch can select at n_h 16 / 32: (kernel variant, H, HW) of the cell, head and
  head weight-gradient kernels in every forward mode, and (ND, more than one 64-row m-tile, row groups) of
  wgrad_kernel.  What the dispatch can select is taken over a universe of layouts that spans the shape envelope.
* ModelLayout accepts the widest observation encoder at the shared-memory limit of each width and refuses 4 gathered
  inputs more.
* wide_n12_h16_ma2c_nc (tests/golden/make_golden_wide_actions.py): the oracle replays the reference's identical agents
  with 12 actions each at n_h = 16 -- initial weights exact, pi / v / R within 1e-5, trained weights within 2e-5.
"""
import hashlib
import itertools

import numpy as np
import pytest

import test_gpu_narrow_widths as nw
from gpu_common import widths
from helpers import golden, load_cfg
from test_hetero_parity import replay, w1_error
from test_wide_actions import OracleIdenticalAgent

NARROW = (16, 32)


def _universe():
    """layouts spanning the envelope at the narrow widths: every agent, chain / grid / cut chain, narrow and wide
    observations, narrow and wide heads (those a width refuses are skipped)"""
    from deeprl_network_b200.layout import ModelLayout
    for v, n_h, topo, n_s, n_a in itertools.product(nw.VARIANTS, NARROW, ('chain8', 'grid5', 'cut8'), (1, 5, 40, 200),
                                                    (1, 4, 8, 15)):
        if v == 'ma2c_ic3' and topo == 'cut8':          # CommNet needs a neighbour (check_model)
            continue
        mask = nw.mask_of(topo)
        try:
            yield ModelLayout(v, widths(v, mask, n_s, n_a), n_a, mask, n_h=n_h, n_fc=n_h, obs_mode='gather')
        except ValueError as e:
            assert 'too wide' in str(e)


@pytest.mark.parametrize('cid', list(nw.CASES))
def test_case_is_in_its_regime(cid):
    c = nw.CASES[cid]
    nw.check_regime(c, nw.layout_of(c))


def test_cases_reach_every_narrow_ffma_instantiation():
    from deeprl_network_b200 import _lib as L
    selectable = set().union(*(nw.instantiations(lay) for lay in _universe()))
    reached = set().union(*(nw.instantiations(nw.layout_of(c)) for c in nw.CASES.values()))
    # the universe is what the dispatch can select: every cell / head instantiation of both widths and head widths ...
    vids = (L.IA2C, L.NC, L.IC3, L.DIAL)
    cells = {('cell_fwd', m, v, h, hw) for m in ('P', 'V', 'PS') for v in vids for h in NARROW for hw in (8, 16)}
    cells |= {('cell_bwd', v, h, hw) for v in vids for h in NARROW for hw in (8, 16)}
    cells |= {(k, h, hw) for k in ('train_heads', 'head_wgrad') for h in NARROW for hw in (8, 16)}
    assert cells <= selectable and len(cells) == 48 + 16 + 8
    # ... and wgrad_kernel at 16 / 32 encoder columns (4 / 2 row groups) past the first m-tile and within it, 64 gate
    # columns (n_h = 16, NeurComm's 64 inputs fill one m-tile) and 128 (n_h = 32, NeurComm's 128 inputs take two)
    wg = {x for x in selectable if x[0] == 'wgrad'}
    assert wg == {('wgrad', 16, False, 4), ('wgrad', 16, True, 4), ('wgrad', 32, False, 2), ('wgrad', 32, True, 2),
                  ('wgrad', 64, False, 1), ('wgrad', 128, False, 1), ('wgrad', 128, True, 1)}
    assert selectable - reached == set()


@pytest.mark.parametrize('n_h', [16, 32, 64])
@pytest.mark.parametrize('variant', ['ma2c_cu', 'ia2c', 'ma2c_nc'])
def test_shared_memory_boundary(variant, n_h):
    """at the widest n_s of the 8-agent chain, ld_in = LD_LIMIT of the width and cell; one more own input moves ld_in
    4 past it (ma2c_cu: 4 more inputs; ia2c / ma2c_nc: 3 gathered ones, padded to 4) and is refused"""
    from deeprl_network_b200.layout import ModelLayout, ffma_fwd_smem_bytes, SMEM_LIMIT
    mask = nw.mask_of('chain8')
    widest = nw.WIDEST.get(n_h, {}).get(variant) or {'ma2c_cu': 744, 'ia2c': 248, 'ma2c_nc': 160}[variant]
    step = 4 if variant == 'ma2c_cu' else 1
    lim = nw.LD_LIMIT[(n_h, variant == 'ma2c_nc')]
    lay = ModelLayout(variant, widths(variant, mask, widest, 4), 4, mask, n_h=n_h, n_fc=n_h, obs_mode='gather')
    assert lay.ld_in == lim and ffma_fwd_smem_bytes(lim, lay.s_dim, n_h) <= SMEM_LIMIT
    assert ffma_fwd_smem_bytes(lim + 4, lay.s_dim, n_h) > SMEM_LIMIT
    with pytest.raises(ValueError, match='%d gathered inputs' % (lim + 4)):
        ModelLayout(variant, widths(variant, mask, widest + step, 4), 4, mask, n_h=n_h, n_fc=n_h, obs_mode='gather')


class _OracleIdenticalNarrow(OracleIdenticalAgent):
    """OracleIdenticalAgent at the fixture's width"""

    def __init__(self, agent, g, mc):
        from oracle import nets
        self.n_s, self.n_a = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']]
        np.random.seed(12)
        self.pol = nets.OraclePolicy(agent, self.n_s, self.n_a[0], g['mask'], n_h=int(g['n_h']), n_fc=int(g['n_h']))
        self.mc, self.N = mc, len(self.n_s)
        self.buf = []


def test_oracle_follows_reference_h16_n12():
    g = golden('wide_n12_h16_ma2c_nc')
    assert int(g['n_h']) == 16 and set(g['n_a_ls'].tolist()) == {12}
    mc = load_cfg('config_ma2c_nc_catchup.ini')['MODEL_CONFIG']
    ag = _OracleIdenticalNarrow('ma2c_nc', g, mc)
    names = [str(n) for n in g['names']]
    assert names == ag.pol.names
    assert tuple(g['w0shape/nc/lstm_comm_0/wx_hid']) == (48, 64) and tuple(g['w0shape/nc/pi_0/w']) == (16, 12)
    for n in names:
        w = np.ascontiguousarray(ag.pol.p[n].detach().numpy())
        assert w.shape == tuple(g['w0shape/' + n]), n
        assert hashlib.sha256(w.tobytes()).hexdigest() == str(g['w0sha/' + n]), n
    trace = replay(g, ag.policy, ag.value, ag.add, ag.backward)
    assert trace.shape == g['trace'].shape
    assert np.abs(trace - g['trace']).max() < 1e-5
    for n in names:
        assert w1_error(g, n, ag.pol.p[n].detach().numpy()) < 2e-5, n
