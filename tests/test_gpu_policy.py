"""GPU: K2-K6 fused forward (message gather, encoders, LSTM cell, heads, sampling) vs the oracle.
Bar (north_star): pi / v within 1e-5 abs in fp32; greedy actions bit-exact; sampled actions identical
for identical uniforms (searchsorted on the float64 cdf like np.random.choice)."""
import numpy as np
import pytest
import torch

from gpu_common import bn, make_pair, nb, obs_dev, oracle_obs, to_dev
from oracle.trainer import OracleTrainer

pytestmark = pytest.mark.gpu
VARIANTS = ['ma2c_nc', 'ma2c_ic3', 'ma2c_dial', 'ia2c', 'ia2c_fp', 'ma2c_cu']
TOL = 1e-5


def _inputs(B, N=8, seed=0, n_s=5, n_a=4):
    rs = np.random.RandomState(seed)
    base = rs.randn(B, N, n_s).astype(np.float32)
    fp = rs.dirichlet(np.ones(n_a), size=(B, N)).astype(np.float32)
    done = (rs.rand(B) < 0.3).astype(np.float32)
    c0 = (rs.randn(B, N, 64) * 0.5).astype(np.float32)
    h0 = np.tanh(rs.randn(B, N, 64)).astype(np.float32) * 0.8
    return rs, base, fp, done, c0, h0


@pytest.mark.parametrize('variant', VARIANTS)
@pytest.mark.parametrize('B', [1, 37, 130, 128, 256])       # 128/256 take the tensor-core path
def test_p_and_v_calls_match_oracle(variant, B):
    from deeprl_network_b200 import _lib as L
    eng, orc, lay, _ = make_pair(variant, B)
    rs, base, fp, done, c0, h0 = _inputs(B)
    eng.set_states(nb(c0), nb(h0))
    orc.states_fw = torch.tensor(np.concatenate([c0, h0], -1))
    obs_d, fp_d, done_d = obs_dev(lay, base), nb(fp), to_dev(done)
    pi_d = torch.zeros(8, B, 4, device='cuda')
    act_d = torch.zeros(8, B, dtype=torch.int32, device='cuda')
    u = rs.rand(B, 8)
    for step in range(3):          # three consecutive steps so the stored state is exercised
        eng.step_p(obs_d, fp_d, done_d, pi_d, act_d, L.SAMPLE_UNIFORM, uniforms=to_dev(np.swapaxes(u, 0, 1), torch.float64))
        pi_o = orc.forward(oracle_obs(lay, base), done, fp, None, 'p')
        np.testing.assert_allclose(bn(pi_d), pi_o, rtol=0, atol=TOL)
        st = bn(eng.get_states_fw())
        np.testing.assert_allclose(st, orc.states_fw.numpy(), rtol=0, atol=TOL)
        # sampled actions: identical to np.random.choice's rule applied to the kernel's own pi
        pk = bn(pi_d)
        exp = np.array([[OracleTrainer.choice(pk[b, i], u[b, i]) for i in range(8)] for b in range(B)])
        np.testing.assert_array_equal(bn(act_d), exp)
        eng.check_tc()
        acts = rs.randint(0, 4, size=(B, 8))
        v_d = torch.zeros(8, B, device='cuda')
        eng.step_v(obs_d, fp_d, done_d, nb(acts).int(), v_d)
        v_o = orc.forward(oracle_obs(lay, base), done, fp, acts, 'v')
        np.testing.assert_allclose(bn(v_d), v_o, rtol=0, atol=TOL)
        np.testing.assert_allclose(bn(eng.get_states_fw()), st, rtol=0, atol=0)      # v-call must not store state
        done = np.zeros(B, dtype=np.float32); done_d = to_dev(done)
        fp = pk.copy(); fp_d = nb(fp)


@pytest.mark.parametrize('variant', VARIANTS)
def test_greedy_actions_bit_exact(variant):
    _greedy_actions_bit_exact(variant, 200)


@pytest.mark.parametrize('variant', VARIANTS)
def test_greedy_actions_bit_exact_tensor_core(variant):
    _greedy_actions_bit_exact(variant, 256)         # whole 128-env tiles: the tensor-core forward samples greedily


def _greedy_actions_bit_exact(variant, B):
    from deeprl_network_b200 import _lib as L
    eng, orc, lay, _ = make_pair(variant, B, scale=1.0)
    assert eng.use_tc == (B % 128 == 0)
    rs, base, fp, done, c0, h0 = _inputs(B, seed=3)
    eng.set_states(nb(c0), nb(h0))
    orc.states_fw = torch.tensor(np.concatenate([c0, h0], -1))
    pi_d = torch.zeros(8, B, 4, device='cuda'); act_d = torch.zeros(8, B, dtype=torch.int32, device='cuda')
    eng.step_p(obs_dev(lay, base), nb(fp), to_dev(done), pi_d, act_d, L.SAMPLE_GREEDY)
    pi_o = orc.forward(oracle_obs(lay, base), done, fp, None, 'p')
    top2 = np.sort(pi_o, axis=-1)
    clear = (top2[..., -1] - top2[..., -2]) > 1e-4              # decisive rows (SURVEY 8c note on ties)
    assert clear.mean() > 0.9
    np.testing.assert_array_equal(bn(act_d)[clear], np.argmax(pi_o, -1)[clear])
    np.testing.assert_array_equal(bn(act_d), np.argmax(bn(pi_d), -1))   # and always argmax of its own pi


def test_philox_sampling_is_deterministic_and_distributed():
    from deeprl_network_b200 import _lib as L
    B = 4096
    eng, orc, lay, _ = make_pair('ma2c_nc', B)
    rs, base, fp, done, c0, h0 = _inputs(B, seed=1)
    base[:] = base[:1]; fp[:] = fp[:1]; done[:] = 1.0              # identical rows -> identical pi
    obs_d, fp_d, done_d = obs_dev(lay, base), nb(fp), to_dev(done)
    pi_d = torch.zeros(8, B, 4, device='cuda'); a1 = torch.zeros(8, B, dtype=torch.int32, device='cuda'); a2 = a1.clone(); a3 = a1.clone()
    eng.reset_states(); eng.step_p(obs_d, fp_d, done_d, pi_d, a1, L.SAMPLE_PHILOX, rng_offset=0)
    eng.reset_states(); eng.step_p(obs_d, fp_d, done_d, pi_d, a2, L.SAMPLE_PHILOX, rng_offset=0)
    eng.reset_states(); eng.step_p(obs_d, fp_d, done_d, pi_d, a3, L.SAMPLE_PHILOX, rng_offset=1)
    assert torch.equal(a1, a2) and not torch.equal(a1, a3)
    p = pi_d[0, 0].cpu().numpy()
    freq = np.bincount(a1[0].cpu().numpy(), minlength=4) / B
    assert np.abs(freq - p).max() < 0.03
    L.check(L.lib().nmarl_rng_advance(L.ptr(eng.rng), 5, L.stream()), 'adv')
    assert eng.rng.cpu().tolist()[1] == 5


def test_grid_topology_forward():
    """5x5 grid (2/3/4 neighbours) NeurComm forward == oracle (cfg5 shape)."""
    from deeprl_network_b200.envs.cacc_env import grid_masks
    mask, _ = grid_masks(5)
    B = 9
    eng, orc, lay, _ = make_pair('ma2c_nc', B, mask=mask)
    rs = np.random.RandomState(0)
    base = rs.randn(B, 25, 5).astype(np.float32); fp = rs.dirichlet(np.ones(4), size=(B, 25)).astype(np.float32)
    c0 = (rs.randn(B, 25, 64) * .5).astype(np.float32); h0 = (rs.rand(B, 25, 64) - .5).astype(np.float32)
    done = np.zeros(B, dtype=np.float32)
    eng.set_states(nb(c0), nb(h0)); orc.states_fw = torch.tensor(np.concatenate([c0, h0], -1))
    pi_d = torch.zeros(25, B, 4, device='cuda')
    eng.step_p(obs_dev(lay, base), nb(fp), to_dev(done), pi_d)
    np.testing.assert_allclose(bn(pi_d), orc.forward(oracle_obs(lay, base), done, fp, None, 'p'), rtol=0, atol=TOL)
    np.testing.assert_allclose(bn(eng.get_states_fw()), orc.states_fw.numpy(), rtol=0, atol=TOL)


def test_missing_buffers_fail_loudly():
    from deeprl_network_b200 import _lib as L
    eng, orc, lay, _ = make_pair('ma2c_nc', 2)
    with pytest.raises(RuntimeError):
        eng.step_p(eng.obs_buf[0], None, eng.done_buf[0], eng.pi_tmp)       # NeurComm needs fingerprints
