"""GPU: the cell kernels across observation widths, action counts and neighbour counts (tests/shape_cases.py), on both
kernel families, against the oracle: p- and v-calls with sampling, the backward pass against float64 autograd, two
optimizer steps -- and everything once more with NaN in the padding columns of the observation rows, which must not
change a single bit (include/nmarl.h: the kernels never read them).

B = 7 and 130 run the FP32-FFMA kernels (130: a ragged third 64-env tile), B = 128 the kernel family the case table
names -- tensor cores up to K = 32, FFMA beyond -- and B = 256 a second 128-env tile.  Tolerances are those of
test_gpu_policy.py / test_gpu_backward.py.  The fused rollout + BPTT path and the other tensor-core instantiations of
some of these shapes are in test_gpu_tc_paths.py.

Gradients are judged as test_gpu_tc_paths.py judges them: an encoder pre-activation that the float64 oracle puts within
1e-5 of 0 may take either sign in fp32, and the share of a gradient entry that hinges on such a unit (RoundoffScale.K)
is not counted as error.  Two shapes have such a unit (one hidden unit of one agent's w_ob / b_ob each); without K
their error is up to 1.0e-5 on gradients of magnitude 5e-4, with it 1e-9."""
import numpy as np
import pytest
import torch

from gpu_common import HP, bn, check_apply_twice, nb, obs_dev, oracle_obs, to_dev
from helpers import random_params
from oracle import nets
from oracle.trainer import OracleTrainer
from shape_cases import CASES, layout_of
from test_gpu_backward import _batch, _oracle_backward
from test_gpu_policy import _inputs
from test_gpu_tc_paths import RoundoffScale

pytestmark = pytest.mark.gpu
TOL = 1e-5
T = 4


def _pair(c, B, dtype):
    from deeprl_network_b200.agents.engine import PolicyEngine
    lay = layout_of(c)
    params = random_params(lay.creation_order(), seed=5, scale=0.3)
    eng = PolicyEngine(lay, B, T, dict(HP), flat_params=lay.pack(params))
    orc = nets.OraclePolicy(c.variant, lay.n_s_ls, c.n_a, lay.mask, params=params, dtype=dtype, n_env=B)
    return eng, orc, lay


def _forward(c, eng, lay, orc, B, poison):
    """Three sampled p-calls + v-calls and a greedy p-call; checked against the oracle when one is given.  Returns every
    output as device tensors."""
    from deeprl_network_b200 import _lib as L
    N, n_a = lay.N, c.n_a
    rs, base, fp, done, c0, h0 = _inputs(B, N=N, seed=2, n_s=max(lay.n_s_ls) if lay.concat else c.n_s, n_a=n_a)
    eng.set_states(nb(c0), nb(h0))
    if orc is not None:
        orc.states_fw = torch.tensor(np.concatenate([c0, h0], -1))
    obs_d, fp_d, done_d = obs_dev(lay, base, poison=poison), nb(fp), to_dev(done)
    assert bool(torch.isnan(obs_d).any()) == (poison and lay.obs_stride > min(lay.n_s_ls if lay.concat else [c.n_s]))
    out = []
    for step in range(4):
        greedy = step == 3
        pi_d = torch.zeros(N, B, n_a, device='cuda')
        act_d = torch.full((N, B), -1, dtype=torch.int32, device='cuda')
        u = rs.rand(B, N)
        if greedy:
            eng.step_p(obs_d, fp_d, done_d, pi_d, act_d, L.SAMPLE_GREEDY)
        else:
            eng.step_p(obs_d, fp_d, done_d, pi_d, act_d, L.SAMPLE_UNIFORM, uniforms=to_dev(np.swapaxes(u, 0, 1), torch.float64))
        eng.check_tc()
        pk, ak, st = bn(pi_d), bn(act_d), bn(eng.get_states_fw())
        acts = rs.randint(0, n_a, size=(B, N))
        v_d = torch.zeros(N, B, device='cuda')
        eng.step_v(obs_d, fp_d, done_d, nb(acts).int(), v_d)
        out += [pi_d, act_d, v_d, eng.get_states_fw()]
        if orc is not None:
            pi_o = orc.forward(oracle_obs(lay, base), done, fp, None, 'p')
            np.testing.assert_allclose(pk, pi_o, rtol=0, atol=TOL)
            np.testing.assert_allclose(st, orc.states_fw.numpy(), rtol=0, atol=TOL)
            if greedy:                                  # first arg-max of its own pi; the oracle's on decisive rows
                np.testing.assert_array_equal(ak, np.argmax(pk, -1))
                top2 = np.sort(pi_o, axis=-1)
                clear = (top2[..., -1] - top2[..., -2]) > 1e-4 if n_a > 1 else np.ones((B, N), bool)
                np.testing.assert_array_equal(ak[clear], np.argmax(pi_o, -1)[clear])
            else:                                       # np.random.choice's rule on the kernel's own pi
                exp = np.array([[OracleTrainer.choice(pk[b, i], u[b, i]) for i in range(N)] for b in range(B)])
                np.testing.assert_array_equal(ak, exp)
            if n_a == 1:
                assert np.all(pk == 1.0) and np.all(ak == 0)
            v_o = orc.forward(oracle_obs(lay, base), done, fp, acts, 'v')
            np.testing.assert_allclose(bn(v_d), v_o, rtol=0, atol=TOL)
            np.testing.assert_array_equal(bn(eng.get_states_fw()), st)          # a v-call must not store state
        done = np.zeros(B, dtype=np.float32); done_d = to_dev(done)
        fp = pk.copy(); fp_d = nb(fp)
    return out


def _load_batch(c, eng, lay, B, poison):
    batch = _batch(eng, lay, T, B, seed=3, N=lay.N, n_s=max(lay.n_s_ls) if lay.concat else c.n_s, n_a=c.n_a, poison=poison)
    mid = B // 2 + 1 if B > 2 else 0
    batch[3][2, mid] = 1                                # one env ends an episode in the middle of the sequence
    eng.done_buf[2, mid] = 1
    assert batch[3][0].sum() == (B + 1) // 2            # and half of them start one
    return batch


def _run(cid, B):
    c = CASES[cid]
    eng, orc32, lay = _pair(c, B, torch.float32)
    assert eng.use_tc == (c.tc and B % 128 == 0), 'the case must run the kernel family it is in the table for'
    # 1. forward
    fwd = _forward(c, eng, lay, orc32, B, poison=False)
    # 2. backward against float64 autograd
    orc = nets.OraclePolicy(c.variant, lay.n_s_ls, c.n_a, lay.mask, params={n: orc32.p[n].detach().numpy() for n in orc32.names},
                            dtype=torch.float64, n_env=B)
    batch = _load_batch(c, eng, lay, B, poison=False)
    kinks = RoundoffScale(orc.p)                        # K: what a ReLU input within 1e-5 of 0 may flip (see there)
    with kinks:
        summ = _oracle_backward(orc, lay, batch)
    eng.backward()
    torch.cuda.synchronize()
    eng.check_tc()
    grads = eng.grads.clone()
    flat = grads.cpu().numpy()
    g = lay.unpack(flat)
    for name in orc.names:
        ref = orc.grads[name].numpy()
        if ref.size == 0:                               # the [0, 64] weights of an agent without neighbours
            continue
        err = np.maximum(np.abs(g[name] - ref) - kinks.K[name].numpy(), 0).max()
        scale = max(1e-3, np.abs(ref).max())
        assert err <= 2e-5 * scale + 1e-7, (name, err, scale)
        if c.n_a == 1 and name.split('/')[-2].startswith('pi'):
            assert np.all(g[name] == 0), (name, 'pi == 1 whatever the logit: exactly zero gradient')
    ls = eng.losses()
    for k in ('policy_loss', 'value_loss', 'entropy_loss'):
        np.testing.assert_allclose(ls[k], summ[k], rtol=1e-4, atol=1e-5, err_msg=k)
    if c.n_a == 1:
        assert np.all(ls['entropy_loss'] == 0)
    pad = np.ones(lay.n_param, bool)
    for _, o, s in lay.entries:
        pad[o:o + int(np.prod(s))] = False
    assert np.all(flat[pad] == 0), 'a float of the flat gradient that belongs to no tensor must be exactly 0'
    # 3. two clip + RMSProp steps (ma2c_cu: with the consensus update)
    check_apply_twice(eng, orc, lay, pad)
    # 4. all of it again on a fresh engine with NaN in the padding columns of every observation row: bit-identical
    eng2, _, _ = _pair(c, B, torch.float32)
    fwd2 = _forward(c, eng2, lay, None, B, poison=True)
    for k, (a, b) in enumerate(zip(fwd, fwd2)):
        assert torch.equal(a, b), 'forward output %d changes with the padding columns of the observation' % k
    _load_batch(c, eng2, lay, B, poison=True)
    eng2.backward()
    assert torch.equal(eng2.grads, grads), 'gradients change with the padding columns of the observation'
    for _ in range(2):
        eng2.apply(1e-2)
    assert torch.equal(eng2.params, eng.params)
    eng2.check_tc()


@pytest.mark.parametrize('B', [7, 130, 128])
@pytest.mark.parametrize('cid', list(CASES))
def test_shape_matches_oracle(cid, B):
    _run(cid, B)


@pytest.mark.parametrize('cid', ['ma2c_nc-chain8-s10-a4', 'ia2c-ladder8-s8-a4', 'ma2c_dial-chain8-s5-a7'])
def test_shape_matches_oracle_two_tensor_core_tiles(cid):
    assert CASES[cid].tc
    _run(cid, 256)
