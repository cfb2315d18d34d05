"""GPU: an agent without neighbours in the homogeneous layout (ModelLayout): the 8-agent chain with agent 3 cut off.

For NeurComm and DIAL such an agent keeps the reference's identical-agent variables: [0, 64] fingerprint / message
weights and real b_fp / b_msg biases (lstm_comm, agents/utils.py:141-156), so the encoder outputs relu(0 + b) still
feed the gate GEMM.  IA2C_FP gets a [0, 64] fcp/w and a real fcp/b; IA2C an observation of its own features only.
No reference fixture covers this case (the CACC configs never cut an agent off); the float64 oracle, which restates
the reference graphs, judges both kernel paths: B = 7 runs the FP32-FFMA kernels, B = 128 the tensor-core ones.

The first half of each of those biases sits at its reference initial value 0, the second half is random.  Where
b <= 0, relu(0 + b) = 0 and TF's ReLU gradient there is 0, so the gradient must be exactly 0; where b > 0 it is the
column sum of the pre-activation gradient.  Every padding float of the flat buffer stays exactly 0 through the
backward and two optimizer steps, and norm_out equals the oracle's norm."""
import numpy as np
import pytest
import torch

from gpu_common import HP, bn, check_apply_twice, cut_chain_mask, nb, oracle_obs, to_dev, widths
from helpers import random_params
from oracle import nets

pytestmark = pytest.mark.gpu
N, CUT, N_A = 8, 3, 4
# the encoder biases of the agent without neighbours whose encoder input is empty
ISO_BIASES = {'ma2c_nc': ['nc/lstm_comm_%d/b_fp', 'nc/lstm_comm_%d/b_msg'], 'ma2c_dial': ['dial/lstm_comm_%d/b_msg'],
              'ia2c': [], 'ia2c_fp': ['lstm_%d/fcp/b']}


def _pair(variant, B, T):
    from deeprl_network_b200.agents.engine import PolicyEngine
    from deeprl_network_b200.layout import ModelLayout
    mask = cut_chain_mask(N, CUT)
    n_s_ls = widths(variant, mask, 5, N_A)
    lay = ModelLayout(variant, n_s_ls, N_A, mask, obs_mode='gather')
    assert lay.nbr[CUT] == [] and all(lay.nbr[i] for i in range(N) if i != CUT)
    params = random_params(lay.creation_order(), seed=6, scale=0.3)
    biases = [n % CUT for n in ISO_BIASES[variant]]
    for n in biases:
        params[n][:len(params[n]) // 2] = 0
    eng = PolicyEngine(lay, B, T, dict(HP), flat_params=lay.pack(params))
    orc = nets.OraclePolicy(variant, n_s_ls, N_A, mask, params=params, dtype=torch.float64, n_env=B)
    return eng, orc, lay, params, biases


@pytest.mark.parametrize('variant', ['ma2c_nc', 'ma2c_dial', 'ia2c', 'ia2c_fp'])
@pytest.mark.parametrize('B', [7, 128])                     # 128: tensor-core path
def test_isolated_agent_matches_oracle(variant, B):
    T = 4
    eng, orc, lay, params, biases = _pair(variant, B, T)
    assert eng.use_tc == (B == 128)
    rs = np.random.RandomState(2)
    base = rs.randn(T, B, N, 5).astype(np.float32)
    fp = rs.dirichlet(np.ones(N_A), size=(T, B, N)).astype(np.float32)
    acts = rs.randint(0, N_A, size=(T, B, N))
    dones = np.zeros((T, B), dtype=np.float32); dones[0, ::2] = 1
    Rs = rs.randn(T, B, N).astype(np.float32); Advs = rs.randn(T, B, N).astype(np.float32)
    c0 = (rs.randn(B, N, 64) * .5).astype(np.float32); h0 = (rs.rand(B, N, 64) - .5).astype(np.float32)
    st = torch.tensor(np.concatenate([c0, h0], -1), dtype=torch.float64)
    # ---- forward p / v ----------------------------------------------------------------------------------------
    eng.set_states(nb(c0), nb(h0))
    orc.states_fw = st.clone()
    obs_d = torch.zeros(N, B, lay.obs_stride, device='cuda'); obs_d[:, :, :5] = nb(base[0])
    pi_d = torch.zeros(N, B, N_A, device='cuda'); v_d = torch.zeros(N, B, device='cuda')
    eng.step_p(obs_d, nb(fp[0]), to_dev(dones[0]), pi_d)
    pi_o = orc.forward(oracle_obs(lay, base[0]), dones[0], fp[0].astype(np.float64), None, 'p')
    np.testing.assert_allclose(bn(pi_d), pi_o, rtol=0, atol=1e-5)
    np.testing.assert_allclose(bn(eng.get_states_fw()), orc.states_fw.numpy(), rtol=0, atol=1e-5)
    eng.step_v(obs_d, nb(fp[0]), to_dev(dones[0]), nb(acts[0]).int(), v_d)
    v_o = orc.forward(oracle_obs(lay, base[0]), dones[0], fp[0].astype(np.float64), acts[0], 'v')
    np.testing.assert_allclose(bn(v_d), v_o, rtol=0, atol=1e-5)
    eng.check_tc()
    # ---- backward ---------------------------------------------------------------------------------------------
    eng.T_cur = T
    eng.obs_buf[:T].zero_(); eng.obs_buf[:T, :, :, :5].copy_(to_dev(np.transpose(base, (0, 2, 1, 3))))
    eng.fp_buf[:T].copy_(to_dev(np.transpose(fp, (0, 2, 1, 3))))
    eng.act_buf[:T].copy_(to_dev(np.transpose(acts, (0, 2, 1)), torch.int32))
    eng.done_buf[:T].copy_(to_dev(dones))
    eng.Rs[:T].copy_(to_dev(np.transpose(Rs, (0, 2, 1)))); eng.Advs[:T].copy_(to_dev(np.transpose(Advs, (0, 2, 1))))
    eng.set_states(nb(c0), nb(h0))
    orc.states_bw, orc.states_fw = st.clone(), st.clone()
    orc.backward([oracle_obs(lay, base[t]) for t in range(T)], fp.astype(np.float64), acts, dones, Rs, Advs, 5e-4,
                 v_coef=HP['v_coef'], e_coef=HP['e_coef'], apply=False)
    eng.backward()
    torch.cuda.synchronize()
    eng.check_tc()
    flat = eng.grads.cpu().numpy()
    gk = lay.unpack(flat)
    for n in orc.names:
        ref = orc.grads[n].numpy()
        if ref.size == 0:                  # the [0, 64] weights of the agent without neighbours
            continue
        err, scale = np.abs(gk[n] - ref).max(), max(1e-3, np.abs(ref).max())
        assert err <= 2e-5 * scale + 1e-7, (n, err, scale)
    for n in biases:
        off = params[n] <= 0
        assert off.sum() >= len(off) // 2 and not off.all()
        assert np.all(gk[n][off] == 0), (n, 'relu(0 + b) with b <= 0 passes no gradient')
        assert np.all(gk[n][~off] != 0), (n, 'b > 0: the column sum of the pre-activation gradient')
    pad = np.ones(lay.n_param, bool)
    for _, o, s in lay.entries:
        pad[o:o + int(np.prod(s))] = False
    assert np.all(flat[pad] == 0)                             # the layout padding gets exactly zero gradient
    check_apply_twice(eng, orc, lay, pad)
