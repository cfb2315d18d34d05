"""GPU: action counts 8 to 15 (the 16-wide head, HW = 16) on both kernel families.

  * the checks of test_gpu_shapes.py on a case table of its own (B = 7 and 130: FFMA; 128 and 256: the family the case
    names): sampled and greedy p-calls and v-calls against the fp32 oracle, backward() against float64 autograd with
    exact zeros on every padding float, two optimizer steps, NaN in the observation padding bit-identical;
  * every tensor-core instantiation and the fused rollout + BPTT path (test_gpu_tc_paths.py), so that 16-wide sv_dlv
    rows written by the rollout are read by BPTT;
  * Philox draws exactly as each kernel's own rule predicts (test_gpu_philox.py);
  * the public agent classes at B = 1 replaying the reference's heterogeneous agents with 2 to 15 actions and its
    identical agents with 12 actions each (tests/golden/wide_*.npz);
  * three rollout + update steps replayed from a CUDA graph equal to the same steps run eagerly, on both families."""
import hashlib
from unittest import mock

import numpy as np
import pytest
import torch

import shape_cases
import test_gpu_philox
import test_gpu_shapes
import test_gpu_tc_paths
from gpu_common import HP, ScriptedEnv, to_dev
from helpers import golden, load_cfg, random_params
from test_hetero_ia2c_parity import replay_agent
from test_hetero_parity import replay, w1_error
from test_wide_actions import FIXTURES, WIDE, agent_of

pytestmark = pytest.mark.gpu

# A subset of test_wide_actions.WIDE that reaches every kernel family and instantiation: the chain for every agent at
# n_a = 8 and 15 (tensor cores up to 15); n_a = 11 for every agent on the grid or the cut chain; the grid at the
# fingerprint boundary (kp_pad 32 / 36 / 44); agents without neighbours on the cut chain.
SHAPES = (['%s-chain8-a%d' % (v, n_a) for v in ('ma2c_nc', 'ma2c_ic3', 'ma2c_dial', 'ia2c', 'ia2c_fp', 'ma2c_cu')
           for n_a in (8, 15)] +
          ['ma2c_nc-grid5-a8', 'ia2c_fp-grid5-a9', 'ma2c_nc-grid5-a11', 'ma2c_dial-grid5-a15', 'ma2c_nc-cut8-a11',
           'ma2c_dial-cut8-a15', 'ma2c_ic3-grid5-a11', 'ia2c-grid5-a11', 'ma2c_cu-cut8-a11', 'ia2c_fp-cut8-a11',
           'ma2c_dial-grid5-a11'])


@pytest.mark.parametrize('B', [7, 130, 128, 256])
@pytest.mark.parametrize('cid', SHAPES)
def test_wide_shape_matches_oracle(cid, B):
    with mock.patch.dict(test_gpu_shapes.CASES, {cid: WIDE[cid]}):
        test_gpu_shapes._run(cid, B)


TC = [pytest.param(dict(variant=v, B=128, T=8, topo='chain8', n_a=15, dones='mixed', kb=None, n_s=5,
                        purpose='n_a = 15: 15 logits + v fill the 16 gate-f staging columns of a column set'),
                   id='n_a15-' + v) for v in ('ma2c_nc', 'ma2c_ic3', 'ma2c_dial', 'ia2c', 'ia2c_fp', 'ma2c_cu')]
TC += [pytest.param(dict(variant='ma2c_nc', B=256, T=8, topo='grid5', n_a=8, dones='mixed', kb=None, n_s=5,
                         purpose='n_a = 8 on the 5x5 grid: kp_pad = 32, the widest fingerprint on tensor cores'),
                    id='n_a8-grid5-ma2c_nc'),
       pytest.param(dict(variant='ma2c_dial', B=128, T=8, topo='chain8cut', n_a=11, dones='mixed', kb=None, n_s=5,
                         purpose='n_a = 11 with an agent without neighbours'), id='n_a11-cut-ma2c_dial')]


@pytest.mark.parametrize('mode', ['unfused', 'fused'])
@pytest.mark.parametrize('c', TC)
def test_wide_tc_paths_match_fp64(c, mode):
    test_gpu_tc_paths.test_tc_paths_match_fp64(c, mode)


@pytest.mark.parametrize('offset', [0, 3])
@pytest.mark.parametrize('B', [37, 256])
@pytest.mark.parametrize('n_a', [8, 15])
@pytest.mark.parametrize('variant', ['ma2c_nc', 'ia2c'])
def test_wide_step_p_draws_the_predicted_actions(variant, n_a, B, offset):
    test_gpu_philox.test_step_p_draws_the_predicted_actions(variant, n_a, B, offset)


@pytest.mark.parametrize('name', FIXTURES)
def test_drop_in_follows_reference_with_wide_heads(name):
    """MA2C_NC / MA2C_DIAL / IA2C_FP at B = 1 (the FFMA kernels) through the reference API: forward, add_transition,
    backward; list returns of unequal length for heterogeneous agents, the identical_agent path for wide_n12_*."""
    from deeprl_network_b200.agents.models import IA2C_FP, MA2C_DIAL, MA2C_NC
    g = golden(name)
    agent, same = agent_of(name), name.startswith('wide_n12_')
    mc = load_cfg('config_ma2c_nc_catchup.ini')['MODEL_CONFIG']
    mc['batch_size'] = str(int(g['n_step']))
    n_s, n_a = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']]
    np.random.seed(12)
    m = {'ma2c_nc': MA2C_NC, 'ma2c_dial': MA2C_DIAL, 'ia2c_fp': IA2C_FP}[agent](
        n_s, n_a, g['mask'], np.zeros_like(g['mask']), -1.0, 10 ** 6, mc, seed=12)
    assert m.identical_agent == same and m.layout.n_a == max(n_a) >= 12
    w0 = m.get_weights()
    names = [str(n) for n in g['names']]
    assert names == [n for n, _ in m.layout.creation_order()]
    for n in names:
        assert hashlib.sha256(np.ascontiguousarray(w0[n]).tobytes()).hexdigest() == str(g['w0sha/' + n]), n
    m.reset()
    if agent == 'ia2c_fp':
        trace = replay_agent(g, agent, m)
    else:
        def policy(ob, d, fp):
            pi = m.forward(ob, d, fp)
            assert [len(p) for p in pi] == n_a
            return pi
        trace = replay(g, policy, lambda ob, d, fp, a: m.forward(ob, d, fp, a, 'v'), m.add_transition,
                       lambda R: m.backward(R, 0))
    assert trace.shape == g['trace'].shape
    assert np.abs(trace - g['trace']).max() < 1e-5
    w1 = m.get_weights()
    for n in names:
        assert w1_error(g, n, w1[n]) < 2e-5, n
    if not same:
        flat = m.engine.params.cpu().numpy()
        assert np.all(flat[m.layout.pi_pad] == np.float32(-1e30))


@pytest.mark.parametrize('B', [128, 64])                      # tensor cores (saving rollout + fused BPTT); FFMA
def test_wide_graph_replay_equals_eager(B):
    """ma2c_nc, n_a = 15: three Philox rollouts + updates, eager and as replays of one captured graph, give the same
    actions and the same parameters bit for bit."""
    from deeprl_network_b200.agents.engine import PolicyEngine
    lay = shape_cases.layout_of(WIDE['ma2c_nc-chain8-a15'])
    flat = lay.pack(random_params(lay.creation_order(), seed=5, scale=0.3))
    T, N = 8, lay.N
    rs = np.random.RandomState(1)
    obs = torch.zeros(T + 1, N, B, lay.obs_stride, device='cuda')
    obs[..., :5] = to_dev(rs.randn(T + 1, N, B, 5).astype(np.float32))
    dones = to_dev((rs.rand(T + 1, B) < 0.1).astype(np.float32))
    outs = []
    for graph in (False, True):
        eng = PolicyEngine(lay, B, T, dict(HP), flat_params=flat, rng_seed=7)
        assert eng.use_tc == (B == 128)
        env = ScriptedEnv(obs, dones)
        eng.obs_buf[0].copy_(obs[0]); eng.done_buf[0].copy_(dones[0])
        eng.lr_dev.fill_(1e-3)
        acts = []

        def one():
            env.t = 0
            eng.rollout(env, sample='philox')
            eng.update(eng.lr_dev)
            eng.normalize_cur()                              # as VecTrainer: a graph replays fixed state buffers
        if graph:                                            # the first update eagerly, the next two from the graph
            one()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                one()
            for _ in range(2):
                g.replay()
        else:
            for _ in range(3):
                one()
                acts.append(eng.act_buf.clone())
        torch.cuda.synchronize()
        eng.check_tc()
        outs.append((eng.params.clone(), acts))
    assert torch.isfinite(outs[0][0]).all()
    assert not torch.equal(outs[0][1][1], outs[0][1][2]), 'each update draws fresh actions'
    assert torch.equal(outs[0][0], outs[1][0])
    assert not torch.equal(outs[0][0], torch.as_tensor(flat, device='cuda'))
