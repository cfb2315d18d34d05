"""CPU: models of up to 128 agents (NMARL_MAX_AGENT).

* ModelLayout / HeteroLayout build all six agents on an 8x8 grid (64 agents) and a 128-vehicle chain, and refuse 129.
* The ctypes mirror of nmarl_model matches the library's struct, and a 128-agent descriptor survives a byte-level
  round trip; the library refuses a 129-agent model or env with a message naming the limit.
* The oracle env replays the many-agent reference fixtures (tests/golden/make_golden_many_agents.py) bit for bit: 61
  vehicles exercise the tail of np.sum's pairwise block, 128 the largest block NumPy sums without recursing.
"""
import ctypes
import glob
import os

import numpy as np
import pytest

from deeprl_network_b200 import _lib as L
from deeprl_network_b200.envs.cacc_env import chain_masks, grid_masks
from deeprl_network_b200.layout import HeteroLayout, ModelLayout
from helpers import GOLDEN, load_cfg
from oracle.cacc import OracleCACC, np_pairwise_sum

VARIANTS = ['ia2c', 'ia2c_fp', 'ma2c_cu', 'ma2c_nc', 'ma2c_ic3', 'ma2c_dial']
FILES = sorted(glob.glob(os.path.join(GOLDEN, 'many*.npz')))
N_A = 4


def _mask(shape):
    return grid_masks(8)[0] if shape == 'grid8x8' else chain_masks(128)[0]


def _layout(variant, mask):
    N = len(mask)
    nm = [int(mask[i].sum()) for i in range(N)]
    n_s_ls = {'ia2c': [5 * (1 + k) for k in nm], 'ia2c_fp': [5 * (1 + k) + N_A * k for k in nm]}.get(variant, [5] * N)
    return ModelLayout(variant, n_s_ls, N_A, mask, obs_mode='gather')


def _hetero(variant, mask):
    rs = np.random.RandomState(len(mask))
    N = len(mask)
    n_a_ls = rs.randint(2, N_A + 1, size=N)
    if variant in ('ia2c', 'ia2c_fp'):        # each agent's own pre-concatenated observation
        n_s_ls = [5 * (1 + int(mask[i].sum())) for i in range(N)]
    else:
        n_s_ls = rs.randint(3, 8, size=N)
    return HeteroLayout(variant, n_s_ls, n_a_ls, mask)


def test_limit_is_128_everywhere():
    assert L.MAX_AGENT == 128
    assert ctypes.sizeof(L.Agent) == 192 and ctypes.sizeof(L.Model) == 48 + 128 * 192 == 24624
    lib = L.lib()
    assert lib.nmarl_sizeof_model() == ctypes.sizeof(L.Model)
    assert lib.nmarl_version() >= 101


@pytest.mark.parametrize('shape', ['grid8x8', 'chain128'])
@pytest.mark.parametrize('variant', VARIANTS)
def test_layouts_accept_up_to_128_agents(variant, shape):
    mask = _mask(shape)
    N = len(mask)
    homo = _layout(variant, mask)
    # 5-feature observations stay on the tensor-core path (narrow encoders) on both graphs
    assert homo.kx_pad <= 32 and homo.kp_pad <= 32
    for lay in (homo, _hetero(variant, mask)):
        assert lay.N == N
        m = lay.c_model()
        assert m.n_agent == N
        # agent-contiguous parameter ranges in order, each agent's neighbours as in the mask
        assert [m.agent[i].p_begin for i in range(1, N)] == [m.agent[i].p_end for i in range(N - 1)]
        assert m.agent[N - 1].p_end <= lay.n_param
        for i in range(N):
            assert [m.agent[i].nbr[s] for s in range(m.agent[i].n_nbr)] == list(np.where(mask[i] == 1)[0])
        # the unpacked reference tensors round-trip through the flat buffer
        flat = lay.init_flat()
        back = lay.pack(lay.unpack(flat))
        np.testing.assert_array_equal(back, flat)


@pytest.mark.parametrize('variant', VARIANTS)
def test_layouts_reject_129_agents(variant):
    mask = chain_masks(129)[0]
    with pytest.raises(ValueError, match='129 > 128'):
        _layout(variant, mask)
    with pytest.raises(ValueError, match='129 > 128'):
        _hetero(variant, mask)


@pytest.mark.parametrize('variant', ['ma2c_nc', 'ma2c_dial', 'ia2c'])
def test_c_model_round_trips_through_ctypes(variant):
    lay = _layout(variant, chain_masks(128)[0])
    m = lay.c_model()
    raw = ctypes.string_at(ctypes.addressof(m), ctypes.sizeof(m))
    m2 = L.Model.from_buffer_copy(raw)
    for f, _ in L.Model._fields_[:-1]:
        assert getattr(m2, f) == getattr(m, f), f
    for i in (0, 1, 63, 126, 127):
        for f, t in L.Agent._fields_:
            a, b = getattr(m.agent[i], f), getattr(m2.agent[i], f)
            assert (list(a) == list(b)) if hasattr(t, '_length_') else a == b, (i, f)
    # the last agent's record is at the end of the struct the library sees
    assert ctypes.addressof(m.agent[127]) - ctypes.addressof(m) == 48 + 127 * 192
    assert m.agent[127].n_nbr == 1 and m.agent[127].nbr[0] == 126 and m.agent[127].p_end == lay.agents_off[127]['p_end']


def test_library_rejects_129_agents():
    lib = L.lib()
    lay = _layout('ma2c_nc', chain_masks(128)[0])
    m = lay.c_model()
    m.n_agent = 129
    a = L.FwdArgs()
    assert lib.nmarl_policy_step_p(ctypes.byref(m), ctypes.byref(a), None) != 0
    assert b'n_agent 129 out of range' in lib.nmarl_last_error()
    cfg = L.CaccCfg()
    cfg.n_agent, cfg.platoon_len = 129, 129
    dummy = ctypes.c_void_p(16)      # never dereferenced: the size check comes first
    assert lib.nmarl_cacc_step(ctypes.byref(cfg), 32, 1, dummy, *([None] * 7), 8, None, None, None, None) != 0
    assert b'129 out of range (1..128)' in lib.nmarl_last_error()


def test_np_sum_order_restated_up_to_128():
    """The device env restates np.sum's 8-accumulator block; it is NumPy's whole algorithm up to 128 values."""
    rs = np.random.RandomState(3)
    for n in (33, 61, 64, 100, 127, 128):
        x = rs.randn(n) * 10.0 ** rs.uniform(-3, 3, n)
        assert np_pairwise_sum(x) == np.sum(x), n


@pytest.mark.parametrize('path', FILES, ids=[os.path.basename(f)[:-4] for f in FILES])
def test_oracle_env_replays_many_agent_fixture(path):
    assert len(FILES) == 6
    g = np.load(path, allow_pickle=True)
    N = int(g['n_vehicle'])
    over = eval(str(g['over']))
    assert over['n_vehicle'] == N
    cp = load_cfg(str(g['ini']), **over)
    env = OracleCACC(cp['ENV_CONFIG'])
    assert env.n_agent == N
    if bool(g['test_mode']):
        env.train_mode = True; env.reset(); env.train_mode = False
        ob = env.reset(test_ind=-1)
    else:
        ob = env.reset()
    assert env.seed == int(g['ep0_seed_after'])
    np.testing.assert_array_equal(env.hs_cur, g['ep0_h0'])
    np.testing.assert_array_equal(env.vs_cur, g['ep0_v0'])
    np.testing.assert_array_equal(np.concatenate(ob), g['ep0_obs'][0])
    acts = g['ep0_acts']
    for t in range(len(acts)):
        ob, r, d, gr = env.step(acts[t])
        assert gr == g['ep0_greward'][t], t
        assert d == bool(g['ep0_done'][t]), t
        np.testing.assert_array_equal(np.broadcast_to(r, (N,)), g['ep0_rew'][t])
        np.testing.assert_array_equal(env.hs_cur, g['ep0_hs'][t])
        np.testing.assert_array_equal(np.concatenate(ob), g['ep0_obs'][t + 1])
    np.testing.assert_array_equal(env.vs_cur, g['ep0_vs_last'])
    np.testing.assert_array_equal(env.us_cur, g['ep0_us_last'])
    # the recorded uniform reproduces the reset (what a batched device env is fed)
    env2 = OracleCACC(cp['ENV_CONFIG'])
    env2.reset(u01=float(g['ep0_u01']))
    np.testing.assert_array_equal(env2.hs_cur, g['ep0_h0'])
    np.testing.assert_array_equal(env2.vs_cur, g['ep0_v0'])
    if str(g['kind']) == 'const0':
        assert g['ep0_done'][-1] and g['ep0_greward'][-1] == -1000.0 * N and len(acts) == 110
        assert np.all(g['ep0_rew'][-1] == -1000.0 * N)          # global reward: every agent gets the sum
