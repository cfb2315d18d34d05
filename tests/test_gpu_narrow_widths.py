"""GPU: num_lstm = 16 and 32 on the FP32-FFMA kernels, crossed with the other axes of the shape envelope.

tests/test_gpu_hidden_width.py runs the narrow widths at one point (the 8-agent chain, n_s = 5, n_a = 4, B <= 128).
Every case here is one of the other axes at n_h 16 or 32, judged against the float64 oracle (oracle/nets.py):
  heads     all six agents, n_a 8 and 15 (the 16-wide head, HW = 16), B = 130: two full 64-row CTAs and a ragged one
  grid      the 5x5 grid (2, 3 and 4 neighbours), n_a = 11: fingerprints of 44 inputs; at 32 the 4-neighbour message
            encoder contracts over 128 inputs, two 64-row m-tiles of wgrad_kernel<32>
  cut       the 8-agent chain with one agent cut off, n_a = 15
  widest    the widest observation encoder ModelLayout accepts at the width (its shared-memory limit), which width 64
            refuses: K > 64 inputs, so wgrad_kernel<16> / <32> runs m-tiles past the first with 4 / 2 row groups
  agents128 a 128-vehicle chain and an 8x8 grid (64 agents), all six agents; IA2C / IA2C_FP clip every agent on its
            own, with 8 / 16 optimizer blocks per agent
  splitk    T x B large enough that the weight-gradient (wgrad_splits) and head weight-gradient (head_splits)
            reductions sum several splits, the last weight-gradient split ending in a ragged 32-row chunk
Each case runs test_gpu_hidden_width._run_against_oracle (p / v forward, backward, the loss terms, exact zeros on the
layout padding, two clip + RMSProp steps) with the gradients judged per tensor and per entry (`judge_grads`), and
asserts the regime it is named after from the layout and the split rules mirrored from csrc/train.cu.
tests/test_narrow_widths.py checks on the host that the table reaches every FFMA instantiation the dispatch can select
at n_h 16 / 32, and the shared-memory boundary of each width.

test_production_shape_ffma runs the shape tools/bench_hidden.py times -- NeurComm catch-up, 4096 envs x 8 agents,
T = 60 -- at n_h 16, 32 and 64 on the FFMA kernels: 32 weight-gradient splits of 7 680 rows, 240 head splits.

test_drop_in_follows_reference_h16_n12 replays tests/golden/wide_n12_h16_ma2c_nc.npz (the reference at num_lstm = 16
with 12 actions per agent) through MA2C_NC at B = 1.
"""
import collections
import hashlib

import numpy as np
import pytest
import torch

import shape_cases
from gpu_common import HP, oracle_obs, to_dev, widths
from helpers import golden, load_cfg, random_params
from oracle import nets
from test_gpu_tc_paths import FLOOR, S_REL, RoundoffScale

pytestmark = pytest.mark.gpu

# ---- the split rules of csrc/train.cu (FFMA path), mirrored ----------------------------------------------------------
RC = 32                                   # rows per wgrad_kernel chunk


def wgrad_splits(R):
    """wgrad_splits: R = T * B reduction rows"""
    return min(max(R // 4096, 1), 32)


def wgrad_rows_per_split(R):
    """wgrad_kernel's `per`: rows per split, a whole number of 32-row chunks; and the rows of the last split"""
    s = wgrad_splits(R)
    per = (-(-R // s) + RC - 1) // RC * RC
    return per, R - (s - 1) * per


def head_splits(R):
    """head_splits"""
    return min(max(R // 1024, 1), 512)


def row_groups(nd):
    """wgrad_kernel<ND>: RG = 256 / (16 * CW / 4) with CW = min(ND, 64)"""
    return 256 // (4 * min(nd, 64))


def opt_blocks(n_groups):
    """nmarl_clip_rmsprop_step: blocks per norm group"""
    return 256 if n_groups == 1 else (32 if n_groups <= 32 else 1024 // n_groups)


def wgrad_jobs(lay):
    """(job, ND, [Ka of every agent]) of each weight-gradient GEMM nmarl_a2c_bptt runs on the FFMA path (run_wgrad)"""
    from deeprl_network_b200 import _lib as L
    H, N, nn = lay.n_h, lay.N, [len(x) for x in lay.nbr]
    jobs = [('gate', 4 * H, [lay.s_dim + H] * N), ('obs', H, [lay._kx(i) for i in range(N)])]
    if lay.vid == L.NC:
        jobs.append(('fp', H, [k * lay.n_a for k in nn]))
    if lay.vid != L.IA2C:
        jobs.append(('msg', H, [H if lay.vid == L.IC3 else k * H for k in nn]))
    if lay.vid == L.DIAL:
        jobs.append(('mfc', H, [H] * N))
    return jobs


def instantiations(lay):
    """The FFMA kernel instantiations one p-call, one v-call and one backward() of the layout launch"""
    from deeprl_network_b200 import _lib as L
    H, HW, vid = lay.n_h, L.head_width(lay.n_a), lay.vid
    out = {('cell_fwd', mode, vid, H, HW) for mode in ('P', 'V', 'PS')}
    out |= {('cell_bwd', vid, H, HW), ('train_heads', H, HW), ('head_wgrad', H, HW)}
    for _, nd, ka in wgrad_jobs(lay):
        out.add(('wgrad', nd, max(ka) > 64, row_groups(nd)))
    return out


# ---- cases -----------------------------------------------------------------------------------------------------------
VARIANTS = ['ia2c', 'ia2c_fp', 'ma2c_cu', 'ma2c_nc', 'ma2c_ic3', 'ma2c_dial']
# the widest own-observation width n_s each variant takes on the 8-agent chain (2 neighbours), by n_h; ld_in of the
# layout sits exactly at the shared-memory limit of the FFMA cell kernel (LD_LIMIT)
WIDEST = {16: {'ma2c_cu': 864, 'ia2c': 288, 'ma2c_nc': 264}, 32: {'ma2c_cu': 824, 'ia2c': 274, 'ma2c_nc': 229}}
LD_LIMIT = {(16, False): 864, (32, False): 824, (64, False): 744, (16, True): 832, (32, True): 760, (64, True): 616}
Case = collections.namedtuple('Case', 'kind variant n_h n_a topo n_s B T')
CASES = collections.OrderedDict()


def _add(kind, variant, n_h, n_a, topo, B, T, n_s=5):
    CASES['%s-%s-h%d-a%d-%s-s%d-B%d-T%d' % (kind, variant, n_h, n_a, topo, n_s, B, T)] = Case(
        kind, variant, n_h, n_a, topo, n_s, B, T)


for _h in (16, 32):
    for _v in VARIANTS:
        for _na in (8, 15):
            _add('heads', _v, _h, _na, 'chain8', 130, 8)
    for _v in ('ma2c_nc', 'ma2c_dial', 'ma2c_ic3', 'ia2c_fp'):
        _add('grid', _v, _h, 11, 'grid5', 70, 8)
    for _v, _ns in WIDEST[_h].items():
        _add('widest', _v, _h, 4, 'chain8', 70, 4, n_s=_ns)
for _v in ('ma2c_nc', 'ma2c_dial', 'ia2c_fp'):
    _add('cut', _v, 16, 15, 'cut8', 130, 8)
for _topo in ('chain128', 'grid8x8'):
    for _v in VARIANTS:
        _add('agents128', _v, 16, 4, _topo, 7, 3)
for _v, _h, _na in (('ma2c_nc', 16, 12), ('ia2c', 16, 15), ('ma2c_dial', 32, 4), ('ma2c_ic3', 32, 4)):
    _add('splitk', _v, _h, _na, 'chain8', 131, 70)


def mask_of(topo):
    if topo in ('chain128', 'grid8x8'):
        from test_gpu_many_agents import _mask
        return _mask(topo)
    return shape_cases.mask_of(topo)


def layout_of(c, n_h=None):
    from deeprl_network_b200.layout import ModelLayout
    mask = mask_of(c.topo)
    n_h = c.n_h if n_h is None else n_h
    return ModelLayout(c.variant, widths(c.variant, mask, c.n_s, c.n_a), c.n_a, mask, n_h=n_h, n_fc=n_h,
                       obs_mode='gather')


def check_regime(c, lay):
    """the regime the case is named after, from its layout and the mirrored split rules"""
    from deeprl_network_b200 import _lib as L
    from deeprl_network_b200.agents.engine import tc_eligible
    assert lay.n_h == c.n_h in (16, 32) and not tc_eligible(lay, c.B)
    jobs = {j: (nd, ka) for j, nd, ka in wgrad_jobs(lay)}
    nn = [len(x) for x in lay.nbr]
    R = c.T * c.B
    if c.kind in ('heads', 'cut', 'grid'):
        assert L.head_width(c.n_a) == 16
    if c.kind == 'heads':
        assert c.B // 64 == 2 and c.B % 64 > 0                        # two full 64-row CTAs, then a ragged one
    if c.kind == 'grid':
        assert sorted(set(nn)) == [2, 3, 4]
        if lay.vid == L.NC:
            assert lay.kp_pad == 44                                     # 4 neighbours x 11 actions
        if c.variant in ('ma2c_nc', 'ma2c_dial', 'ia2c_fp') and c.n_h == 32:
            assert max(jobs['msg'][1]) == 128 and jobs['msg'][0] == 32   # two m-tiles of wgrad_kernel<32>
    if c.kind == 'cut':
        assert nn.count(0) == 1
    if c.kind == 'widest':
        nd, ka = jobs['obs']
        assert max(ka) > 64 and row_groups(nd) == {16: 4, 32: 2}[c.n_h]
        assert lay.ld_in == LD_LIMIT[(c.n_h, lay.s_dim == 3 * c.n_h)]
        with pytest.raises(ValueError, match='too wide'):
            layout_of(c, n_h=64)
    if c.kind == 'agents128':
        assert lay.N == {'chain128': 128, 'grid8x8': 64}[c.topo]
        if c.variant in ('ia2c', 'ia2c_fp'):
            assert opt_blocks(lay.N) == 1024 // lay.N < 32           # 8 / 16 optimizer blocks per agent
    if c.kind == 'splitk':
        per, last = wgrad_rows_per_split(R)
        assert wgrad_splits(R) > 1 and head_splits(R) > 1 and 0 < last < per and last % RC > 0


# ---- gradient judgement ------------------------------------------------------------------------------------------------
def judge_grads(tag, gk, g64, S, K):
    """Per tensor: max(|g - g64| - K, 0) within 2e-5 max(1e-3, max|g64|) + 1e-7 (K: what a ReLU kink may flip, see
    RoundoffScale).  Per entry: that error over the entry's float64 round-off scale S (floored at S_REL of the tensor's
    largest) within FLOOR, so a few wrong lanes cannot hide behind the largest entry of their tensor.  Returns the
    worst (ratio, tensor) of both."""
    tensor, entry = {}, {}
    for n, ref in g64.items():
        if ref.size == 0:                  # the [0, n_h] fingerprint / message weights of an agent without neighbours
            continue
        err = np.maximum(np.abs(gk[n] - ref) - K[n], 0)
        scale = max(1e-3, np.abs(ref).max())
        assert err.max() <= 2e-5 * scale + 1e-7, (tag, n, err.max(), scale)
        tensor[n] = float(err.max() / scale)
        entry[n] = float((err / np.maximum(S[n], S_REL * S[n].max() + 1e-300)).max())
    wt, we = max(tensor, key=tensor.get), max(entry, key=entry.get)
    print('[%s] worst per-tensor error / max|g| %.2e (%s), worst per-entry error / S %.2e (%s)' % (
        tag, tensor[wt], wt, entry[we], we))
    bad = sorted(((r, n) for n, r in entry.items() if r > FLOOR), reverse=True)
    assert not bad, (tag, 'per-entry error / round-off scale', bad[:6])
    return (tensor[wt], wt), (entry[we], we)


class Judge:
    """test_gpu_hidden_width._run_against_oracle's gradient check: RoundoffScale around the oracle's backward"""

    def mode(self, orc):
        self.rs = RoundoffScale(orc.p)
        return self.rs

    def check(self, tag, gk, orc):
        judge_grads(tag, gk, {n: orc.grads[n].numpy() for n in orc.names}, {n: self.rs.S[n].numpy() for n in orc.names},
                    {n: self.rs.K[n].numpy() for n in orc.names})


@pytest.mark.parametrize('cid', list(CASES))
def test_narrow_width_case_matches_fp64(cid):
    from deeprl_network_b200.agents.engine import PolicyEngine
    from test_gpu_hidden_width import _run_against_oracle
    c = CASES[cid]
    lay = layout_of(c)
    check_regime(c, lay)
    T, B, N, n_a = c.T, c.B, lay.N, c.n_a
    params = random_params(lay.creation_order(), seed=3, scale=0.3)
    orc = nets.OraclePolicy(c.variant, lay.n_s_ls, n_a, lay.mask, n_h=c.n_h, n_fc=c.n_h, params=params,
                            dtype=torch.float64, n_env=B)
    eng = PolicyEngine(lay, B, T, dict(HP), flat_params=lay.pack(params))
    assert eng.use_tc is False and eng.wpack is None
    rs = np.random.RandomState(4)
    base = rs.randn(T, B, N, c.n_s).astype(np.float32)
    fp = rs.dirichlet(np.ones(n_a), size=(T, B, N)).astype(np.float32)
    acts = rs.randint(0, n_a, size=(T, B, N))
    dones = np.zeros((T, B), dtype=np.float32); dones[0, ::2] = 1; dones[T // 2, 1::3] = 1
    Rs = rs.randn(T, B, N).astype(np.float32); Advs = rs.randn(T, B, N).astype(np.float32)
    obs_o = [oracle_obs(lay, base[t]) for t in range(T)]
    base_dev = torch.zeros(T, N, B, lay.obs_stride, device='cuda')
    base_dev[..., :c.n_s] = to_dev(np.transpose(base, (0, 2, 1, 3)))
    _run_against_oracle(cid, eng, orc, lay, c.n_h, obs_o, base_dev, fp, acts, dones, Rs, Advs, judge=Judge())
    assert eng.norm_out.numel() == (N if c.variant in ('ia2c', 'ia2c_fp') else 1)


# ---- the shape tools/bench_hidden.py times ---------------------------------------------------------------------------
PROD_B, PROD_CHUNK = 4096, 512


@pytest.mark.parametrize('n_h', [16, 32, 64])
def test_production_shape_ffma(n_h):
    """NeurComm catch-up, 4096 envs x 8 agents, T = 60, FFMA kernels: one rollout through CACCEnv, the n-step returns
    against float64, backward against float64 autograd accumulated over env chunks (the loss is a mean over (t, env),
    so chunk gradients -- and their round-off scales -- add up with weight chunk / B), then the optimizer step."""
    from deeprl_network_b200.agents.engine import PolicyEngine
    from deeprl_network_b200.envs.cacc_env import CACCEnv
    from deeprl_network_b200.layout import ModelLayout
    B, chunk = PROD_B, PROD_CHUNK
    cp = load_cfg('config_ma2c_nc_catchup.ini', n_env=B)
    env = CACCEnv(cp['ENV_CONFIG'])
    mc = cp['MODEL_CONFIG']
    N, mask, T = env.n_agent, env.neighbor_mask, mc.getint('batch_size')
    R = T * B
    assert (N, T) == (8, 60) and wgrad_splits(R) == 32 and wgrad_rows_per_split(R) == (7680, 7680)
    assert head_splits(R) == 240
    lay = ModelLayout('ma2c_nc', env.n_s_ls, 4, mask, n_h=n_h, n_fc=n_h, obs_mode='gather')
    params = random_params(lay.creation_order(), seed=1, scale=0.3)
    hp = dict(v_coef=mc.getfloat('value_coef'), e_coef=mc.getfloat('entropy_coef'), max_grad_norm=mc.getfloat('max_grad_norm'),
              alpha=mc.getfloat('rmsp_alpha'), epsilon=mc.getfloat('rmsp_epsilon'), gamma=mc.getfloat('gamma'),
              reward_norm=mc.getfloat('reward_norm'), reward_clip=mc.getfloat('reward_clip'))
    e = PolicyEngine(lay, B, T, hp, flat_params=lay.pack(params), distance_mask=env.distance_mask,
                     coop_gamma=env.coop_gamma, use_tc=False)
    assert not e.use_tc
    dev = env.device
    rs = np.random.RandomState(5)
    env.reset_device(u01=torch.as_tensor(rs.rand(N // env.platoon_len, B)).to(dev))
    e.begin_episode(env)
    c0 = (rs.randn(N, B, n_h) * 0.5).astype(np.float32)
    h0 = (np.tanh(rs.randn(N, B, n_h)) * 0.8).astype(np.float32)
    e.set_states(torch.as_tensor(c0).to(dev), torch.as_tensor(h0).to(dev))
    e.done_buf[0].copy_(torch.as_tensor((rs.rand(B) < 0.5).astype(np.float32)).to(dev))
    e.rollout(env, sample='uniform', uniforms=torch.as_tensor(rs.rand(T + 1, N, B)).to(dev))
    e.compute_returns()
    torch.cuda.synchronize()
    obs = e.obs_buf.cpu().numpy()[..., :5]          # [T+1, N, B, 5]
    fp = e.fp_buf.cpu().numpy()                      # [T+1, N, B, 4]
    dones = e.done_buf.cpu().numpy()                 # [T+1, B] (slot t = done before step t)
    acts = e.act_buf.cpu().numpy()                   # [T, N, B]
    vals, grew = e.val_buf.cpu().numpy(), e.grew_buf.cpu().numpy()
    Rs, Advs, R_end = e.Rs.cpu().numpy(), e.Advs.cpu().numpy(), e.R_end.cpu().numpy()
    assert 0 < dones[0].sum() < B                     # half the envs start the batch with a fresh state
    # n-step returns / advantages in float64 over the whole batch
    assert env.coop_gamma < 0
    Rf = np.where(dones[T][None, :] != 0, 0.0, R_end.astype(np.float64))
    for t in range(T - 1, -1, -1):
        Rf = grew[t][None, :] / hp['reward_norm'] + hp['gamma'] * Rf * (1.0 - dones[t + 1][None, :])
        assert np.abs(Rs[t] - Rf).max() < 1e-5, ('R', t)
        assert np.abs(Advs[t] - (Rf - vals[t])).max() < 2e-5, ('Adv', t)
    # backward against float64 autograd, accumulated over env chunks
    e.backward()
    torch.cuda.synchronize()
    g_k = lay.unpack(e.grads.cpu().numpy())
    st0 = np.concatenate([np.swapaxes(c0, 0, 1), np.swapaxes(h0, 0, 1)], -1)
    g64 = S = K = None
    for lo in range(0, B, chunk):
        sl = slice(lo, lo + chunk)
        oc = nets.OraclePolicy('ma2c_nc', env.n_s_ls, 4, mask, n_h=n_h, n_fc=n_h, params=params, dtype=torch.float64,
                               n_env=chunk)
        oc.states_bw = torch.tensor(st0[sl], dtype=torch.float64)
        mode = RoundoffScale(oc.p)
        with mode:
            oc.backward([[obs[t, i, sl] for i in range(N)] for t in range(T)], np.transpose(fp[:T, :, sl], (0, 2, 1, 3)),
                        np.transpose(acts[:, :, sl], (0, 2, 1)), dones[:T, sl], np.transpose(Rs[:, :, sl], (0, 2, 1)),
                        np.transpose(Advs[:, :, sl], (0, 2, 1)), 5e-4, v_coef=hp['v_coef'], e_coef=hp['e_coef'],
                        apply=False)
        w = chunk / B
        parts = [{n: d[n].numpy() * w for n in oc.names} for d in (oc.grads, mode.S, mode.K)]
        g64, S, K = parts if g64 is None else [{n: a[n] + p[n] for n in p} for a, p in zip((g64, S, K), parts)]
        del oc, mode
    judge_grads('production n_h=%d B=%d T=%d' % (n_h, B, T), g_k, g64, S, K)
    # clip + RMSProp on the oracle's gradient against the kernel's parameters
    oa = nets.OraclePolicy('ma2c_nc', env.n_s_ls, 4, mask, n_h=n_h, n_fc=n_h, params=params, dtype=torch.float64, n_env=1)
    oa.grads = {n: torch.tensor(g64[n]) for n in oa.names}
    norms = oa.apply_grads(5e-4, hp['max_grad_norm'], hp['alpha'], hp['epsilon'])
    e.apply(5e-4)
    torch.cuda.synchronize()
    np.testing.assert_allclose(e.norm_out.cpu().numpy(), norms, rtol=2e-4)
    w = lay.unpack(e.params.cpu().numpy())
    for n in oa.names:
        np.testing.assert_allclose(w[n], oa.p[n].detach().numpy(), rtol=0, atol=3e-6, err_msg=n)


# ---- the reference at num_lstm = 16 with 12 actions ------------------------------------------------------------------
def test_drop_in_follows_reference_h16_n12():
    """MA2C_NC at B = 1 (FFMA, n_h = 16, HW = 16) replays wide_n12_h16_ma2c_nc through the reference API: the initial
    weights bit for bit, every pi / v / R within 1e-5, the trained weights' sample within 2e-5."""
    from deeprl_network_b200.agents.models import MA2C_NC
    from test_hetero_parity import replay, w1_error
    g = golden('wide_n12_h16_ma2c_nc')
    mc = load_cfg('config_ma2c_nc_catchup.ini')['MODEL_CONFIG']
    mc['batch_size'] = str(int(g['n_step']))
    mc['num_lstm'] = mc['num_fc'] = str(int(g['n_h']))
    n_s, n_a = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']]
    np.random.seed(12)
    m = MA2C_NC(n_s, n_a, g['mask'], np.zeros_like(g['mask']), -1.0, 10 ** 6, mc, seed=12)
    assert m.identical_agent and m.layout.n_h == 16 and m.layout.n_a == 12 and not m.engine.use_tc
    w0 = m.get_weights()
    names = [str(n) for n in g['names']]
    assert names == [n for n, _ in m.layout.creation_order()]
    for n in names:
        assert hashlib.sha256(np.ascontiguousarray(w0[n]).tobytes()).hexdigest() == str(g['w0sha/' + n]), n
    m.reset()
    trace = replay(g, lambda ob, d, fp: m.forward(ob, d, fp), lambda ob, d, fp, a: m.forward(ob, d, fp, a, 'v'),
                   m.add_transition, lambda R: m.backward(R, 0))
    assert trace.shape == g['trace'].shape
    assert np.abs(trace - g['trace']).max() < 1e-5
    w1 = m.get_weights()
    for n in names:
        assert w1_error(g, n, w1[n]) < 2e-5, n
