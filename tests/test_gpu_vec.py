"""GPU: the batched (n_env > 1) device-resident loop.  (1) a B-env rollout equals B independent
single-env oracle rollouts fed the same uniforms; (2) its gradient equals the oracle's batched
autograd on the recorded trajectories; (3) CUDA-graph replay == eager execution; (4) throughput-mode
auto-reset keeps episodes independent."""
import numpy as np
import pytest
import torch

from helpers import CFG, load_cfg
from oracle import nets
from oracle.buffers import nstep_returns
from oracle.cacc import OracleCACC
from oracle.trainer import OracleTrainer

pytestmark = pytest.mark.gpu


def _make(agent, B, graph=False, sample='philox', **over):
    from deeprl_network_b200.agents.models import IA2C, IA2C_CU, IA2C_FP, MA2C_DIAL, MA2C_IC3, MA2C_NC
    from deeprl_network_b200.envs.cacc_env import CACCEnv
    from deeprl_network_b200.utils import VecTrainer
    cls = {'ma2c_nc': MA2C_NC, 'ia2c': IA2C, 'ma2c_ic3': MA2C_IC3, 'ma2c_dial': MA2C_DIAL, 'ia2c_fp': IA2C_FP,
           'ma2c_cu': IA2C_CU}[agent]
    cp = load_cfg(CFG[agent], n_env=B, **over)
    env = CACCEnv(cp['ENV_CONFIG'])
    kw = dict(obs_mode='gather') if agent == 'ia2c' else {}
    model = cls(env.n_s_ls, env.n_a_ls, env.neighbor_mask, env.distance_mask, env.coop_gamma, 10 ** 6,
                cp['MODEL_CONFIG'], seed=12, n_env=B, **kw)
    return cp, env, model, VecTrainer(env, model, graph=graph, sample=sample)


def _n_s(agent, oenv):
    """IA2C_FP counts the attached fingerprints in the state width (agents/models.py:172-177)."""
    if agent != 'ia2c_fp':
        return oenv.n_s_ls
    return [n + 4 * int(np.sum(oenv.neighbor_mask[i])) for i, n in enumerate(oenv.n_s_ls)]


@pytest.mark.parametrize('agent', ['ma2c_nc', 'ma2c_ic3', 'ma2c_dial', 'ia2c', 'ia2c_fp', 'ma2c_cu'])
def test_batched_rollout_and_update_vs_oracle(agent):
    B = 5
    cp, env, model, vt = _make(agent, B, sample='uniform')
    e = model.engine
    T, N = e.T, e.N
    rs = np.random.RandomState(3)
    u0 = rs.rand(1, B)
    uni = rs.rand(T + 1, N, B)
    env.reset_device(u01=torch.as_tensor(u0).to(env.device))
    e.reset_states(); e.begin_episode(env)
    w0 = model.get_weights()
    e.rollout(env, sample='uniform', uniforms=torch.as_tensor(uni).to(env.device))
    e.compute_returns()
    torch.cuda.synchronize()
    acts = e.act_buf.cpu().numpy(); vals = e.val_buf.cpu().numpy(); grew = e.grew_buf.cpu().numpy()
    Rs = e.Rs.cpu().numpy(); Advs = e.Advs.cpu().numpy(); R_end = e.R_end.cpu().numpy()
    mask = env.neighbor_mask
    g = lambda k: float(cp['MODEL_CONFIG'][k])
    obs_rec = [[None] * B for _ in range(T)]
    for b in range(B):
        oenv = OracleCACC(cp['ENV_CONFIG']); ob = oenv.reset(u01=u0[0, b])
        pol = nets.OraclePolicy(agent, _n_s(agent, oenv), 4, mask, params=w0)
        done, fp = True, np.ones((N, 4)) / 4
        rews, vs, dones = [], [], []
        for t in range(T):
            obs_rec[t][b] = ob
            pi = pol.forward(ob, done, fp[None], None, 'p')[0]
            a = np.array([OracleTrainer.choice(pi[i], uni[t, i, b]) for i in range(N)])
            np.testing.assert_array_equal(acts[t, :, b], a)
            v = pol.forward(ob, done, fp[None], a[None], 'v')[0]
            np.testing.assert_allclose(vals[t, :, b], v, rtol=0, atol=1e-5)
            fp = pi
            oenv.update_fingerprint(pi)
            ob, r, done, gr = oenv.step(a)
            assert abs(grew[t, b] - gr) <= 1e-9 * abs(gr)
            rews.append(np.broadcast_to(np.asarray(r) / g('reward_norm'), (N,))); vs.append(v); dones.append(done)
        pi2 = pol.forward(ob, done, fp[None], None, 'p')[0]
        a2 = np.array([OracleTrainer.choice(pi2[i], uni[T, i, b]) for i in range(N)])
        Re = np.zeros(N) if done else pol.forward(ob, done, fp[None], a2[None], 'v')[0]
        if not done:
            np.testing.assert_allclose(R_end[:, b], Re, rtol=0, atol=1e-5)
        oR, oA = nstep_returns(np.array(rews), np.array(vs), dones, Re, g('gamma'), env.coop_gamma, env.distance_mask)
        np.testing.assert_allclose(Rs[:, :, b].T, oR, rtol=0, atol=1e-5)
        np.testing.assert_allclose(Advs[:, :, b].T, oA, rtol=0, atol=2e-5)
    # batched gradient on the recorded trajectories (oracle consumes the kernel's own Rs / Advs)
    pol = nets.OraclePolicy(agent, _n_s(agent, OracleCACC(cp['ENV_CONFIG'])), 4, mask, params=w0, n_env=B, dtype=torch.float64)
    obs_t = [[np.stack([obs_rec[t][b][i] for b in range(B)]) for i in range(N)] for t in range(T)]
    fp_t = np.transpose(e.fp_buf[:T].cpu().numpy(), (0, 2, 1, 3))
    dones_t = e.done_buf[:T].cpu().numpy()
    s = pol.backward(obs_t, fp_t, np.transpose(acts, (0, 2, 1)), dones_t, np.transpose(Rs, (0, 2, 1)),
                     np.transpose(Advs, (0, 2, 1)), 5e-4, v_coef=g('value_coef'), e_coef=g('entropy_coef'), apply=False)
    e.backward(); torch.cuda.synchronize()
    gr = model.layout.unpack(e.grads.cpu().numpy())
    for name in pol.names:
        ref = pol.grads[name].numpy()
        assert np.abs(gr[name] - ref).max() <= 5e-5 * max(1e-3, np.abs(ref).max()) + 1e-7, name


def test_graph_replay_equals_eager():
    _graph_replay_equals_eager('ma2c_nc', 16)


@pytest.mark.parametrize('agent', ['ma2c_nc', 'ma2c_ic3', 'ma2c_dial', 'ia2c', 'ia2c_fp', 'ma2c_cu'])
def test_graph_replay_equals_eager_tensor_core(agent):
    """B = 128: the captured graph replays the tensor-core update (saved rollout + fused BPTT) that bench.py times."""
    _graph_replay_equals_eager(agent, 128)


def _graph_replay_equals_eager(agent, B):
    outs = []
    for graph in (False, True):
        cp, env, model, vt = _make(agent, B, graph=graph)
        assert model.engine.use_tc == (B % 128 == 0)
        vt.start()
        for _ in range(3):
            vt.update()
        torch.cuda.synchronize()
        model.engine.check_tc()
        outs.append((model.engine.params.clone(), model.engine.grew_buf.clone(), env.t_dev.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2])


def test_auto_reset_of_finished_envs():
    cp, env, model, vt = _make('ma2c_ic3', 64)
    vt.start()
    seen_reset = False
    for k in range(12):
        vt.update()
        t = env.t_dev.cpu().numpy()
        assert np.all(t % 60 == 0) and t.max() <= 600
        if len(np.unique(t)) > 1:
            seen_reset = True
            fresh = t == 0
            assert torch.all(model.engine.done_buf[0, torch.as_tensor(fresh).cuda()] == 1)
            assert torch.all(model.engine.h[model.engine.cur][:, torch.as_tensor(fresh).cuda()] == 0)
    assert seen_reset                      # random policies collide early in some envs
    assert np.isfinite(model.engine.params.cpu().numpy()).all()


@pytest.mark.parametrize('agent', ['ma2c_nc', 'ma2c_dial'])
def test_training_forward_reproduces_saved_rollout(agent):
    """Tensor-core path, one batch: the separate training forward (nmarl_a2c_backward) re-runs the rollout's cell
    steps from states_bw and saves the same activations, so BPTT gives the saved rollout's gradient and loss partials
    bit for bit."""
    cp, env, model, vt = _make(agent, 128, sample='uniform')
    e = model.engine
    assert e.use_tc and e.fuse_save
    rs = np.random.RandomState(0)
    env.reset_device(u01=torch.as_tensor(rs.rand(1, 128)).to(env.device))
    e.reset_states(); e.begin_episode(env)
    uni = torch.as_tensor(rs.rand(e.T + 1, e.N, 128)).to(env.device)
    e.rollout(env, sample='uniform', uniforms=uni)
    assert e.saved_rollout
    e.compute_returns()
    e.backward()                                 # nmarl_a2c_bptt on the rollout's saved activations
    torch.cuda.synchronize()
    fused = (e.grads.clone(), e.loss_part.clone())
    assert not e.saved_rollout
    e.h_bw.copy_(e.h_seq[0]); e.c_bw.copy_(e.c_seq[0])
    e.backward()                                 # nmarl_a2c_backward: training forward + BPTT on the same buffers
    e.check_tc()
    torch.cuda.synchronize()
    assert torch.equal(fused[0], e.grads)
    assert torch.equal(fused[1], e.loss_part)


@pytest.mark.parametrize('agent', ['ma2c_nc', 'ma2c_dial'])
def test_saved_rollout_equals_separate_training_forward(agent):
    """Tensor-core path over two updates: activations saved by the rollout p-calls give the same gradients,
    parameters and loss terms, bit for bit, as the reference-style separate training forward (same inputs and
    weights, the same heads kernel)."""
    grads = []
    for fuse in (True, False):
        cp, env, model, vt = _make(agent, 128, sample='uniform')
        e = model.engine
        assert e.use_tc
        e.fuse_save = fuse
        rs = np.random.RandomState(0)
        env.reset_device(u01=torch.as_tensor(rs.rand(1, 128)).to(env.device))
        e.reset_states(); e.begin_episode(env)
        uni = torch.as_tensor(rs.rand(e.T + 1, e.N, 128)).to(env.device)
        for _ in range(2):                      # second batch starts from a non-zero LSTM state
            e.rollout(env, sample='uniform', uniforms=uni)
            assert e.saved_rollout == fuse
            e.compute_returns(); e.backward(); e.apply(5e-4); e.roll_buffers()
        e.check_tc()
        torch.cuda.synchronize()
        grads.append((e.grads.clone(), e.params.clone(), e.act_buf.clone(), torch.tensor(e.losses()['policy_loss'])))
    for k in range(4):
        assert torch.equal(grads[0][k], grads[1][k])
