"""GPU: both modes of the tensor-core training step against one float64 oracle per case and mode.

The LSTM state layout follows from the variant (feature-major, DIAL env-major), and the training forward either runs
in `backward()` on recorded buffers (unfused) or is saved by the rollout p-calls and folded into the BPTT call (fused:
`rollout(sample='uniform')` on a scripted env, then `backward()`).  Each case runs in both modes, as separate
parameter sets; one set of inputs and a float64 oracle (oracle/nets.py autograd) of the trajectory the mode ran judge
pi / v / states, the loss terms, every gradient, and zero gradient on the layout padding.

Gradients are judged per entry as well as per tensor.  A weight used as x @ W gets the round-off scale
S_W = sum over its uses of |x|^T |delta| (delta = the gradient of the product), a bias S_b = sum |delta|; both are
collected from the oracle's own backward.  The tensor-core error max|g - g64| / S of a tensor must stay within 4x that
of the FP32-FFMA kernels (use_tc=False) on the same buffers plus FLOOR, so a few wrong lanes cannot hide behind the
largest entry of their tensor.
"""
import numpy as np
import pytest
import torch
from torch.overrides import TorchFunctionMode

from gpu_common import HP, ScriptedEnv, ladder_masks, nb, oracle_obs, to_dev, widths
from helpers import golden, random_params
from oracle import nets
from oracle.cacc import chain_masks

pytestmark = pytest.mark.gpu

# Per-entry ratio floor, set from the unmutated kernels on an H100 SXM (80 GB): the worst tensor-core ratio over all
# cases is 2.6e-5 (nc/lstm_comm_1/wx_hid in the T = 160..168 NeurComm cases, where ReLU kinks of the message encoder
# reach wx_hid through BPTT); every T = 8 case stays below 1e-5.  A lost segment or partial sum, or a dropped lo term,
# is orders of magnitude above it.
FLOOR = 4e-5
# Entries whose scale is below S_REL x the largest of their tensor are judged against that level instead: there one
# product dominates and the fp32 error of delta itself (1 - sigmoid near saturation, cancellation in dz) is no longer
# small next to S, for the FFMA kernels as much as for the tensor-core ones.
S_REL = 1e-3
# ReLU inputs closer to 0 than this may take either sign in fp32 (see RoundoffScale.K)
KINK = 1e-5
NH = 64

# ---- mirror of the weight-gradient split (csrc/tc_wgrad.cu): a case asserts the regime it is named after ---------
SEG_KB = 20                     # k-blocks accumulated in registers before the accumulator is drained


def wgrad_splits(n_agent):
    """nmarl_tc_wgrad_splits"""
    s = 33
    while 4 * s * n_agent > 132 * 8 and s > 1:
        s = (s + 1) // 2
    return s


def wgrad_kb_per_split(B, T, n_agent):
    """32-row k-blocks per split, and the k-blocks of the last split (0: idle)"""
    total, splits = T * B // 32, wgrad_splits(n_agent)
    per = -(-total // splits)
    return per, max(0, total - (splits - 1) * per)


# ---- cases ---------------------------------------------------------------------------------------------------------
VARIANTS = ['ma2c_nc', 'ma2c_ic3', 'ma2c_dial', 'ia2c', 'ia2c_fp', 'ma2c_cu']
CASES = []


CUT = 3                         # topo 'chain8cut': the agent without neighbours


def _case(cid, variant, B, T, purpose, topo='chain8', n_a=4, dones='mixed', kb=None, n_s=5):
    CASES.append(pytest.param(dict(variant=variant, B=B, T=T, topo=topo, n_a=n_a, dones=dones, kb=kb, purpose=purpose,
                              n_s=n_s), id=cid))


for _v in VARIANTS:
    _case('variant-' + _v, _v, 256, 8, 'every variant on the 8-agent chain, two 128-env tiles')
for _v in ('ma2c_nc', 'ma2c_ic3', 'ma2c_dial'):
    _case('hetero-' + _v, _v, 256, 8, 'unequal n_s / n_a on an irregular graph (tests/golden/hetero_*)', topo='hetero')
for _v in ('ma2c_nc', 'ma2c_dial'):
    _case('hetero-iso-' + _v, _v, 256, 8, 'unequal n_s / n_a, the last agent without neighbours: no fingerprint / '
          'message k-blocks (tests/golden/hetero_iso_*)', topo='hetero_iso')
for _v in ('ma2c_nc', 'ia2c_fp'):
    _case('isolated-' + _v, _v, 256, 8, '8-agent chain with agent %d cut off: [0, 64] fingerprint / message weights '
          'and non-zero b_fp / b_msg' % CUT, topo='chain8cut')
for _v in ('ma2c_nc', 'ma2c_ic3'):
    _case('done-t0-' + _v, _v, 256, 8, 'every env done at t = 0: the non-zero initial state is masked out', dones='t0')
    _case('done-block-' + _v, _v, 256, 8, 'one whole 32-row block (one gate-bias partial) done mid-sequence',
          dones='block')
    _case('done-cta-' + _v, _v, 256, 8, 'rows 63 and 64 done: the boundary between two 64-row CTAs', dones='cta')
    _case('done-all-' + _v, _v, 256, 8, 'every env done at one step mid-sequence', dones='all')
for _v in ('ma2c_nc', 'ma2c_dial', 'ma2c_ic3', 'ia2c'):
    _case('grid5x5-' + _v, _v, 128, 8, '5x5 grid: 2, 3 and 4 neighbours (DIAL m64n192 / m64n256 message wgrad)',
          topo='grid5')
_case('agents32-ma2c_nc', 'ma2c_nc', 128, 8, '32-agent chain (NMARL_MAX_AGENT): 5 weight-gradient splits', topo='chain32')
for _na in (2, 7):
    for _v in ('ma2c_nc', 'ia2c'):
        _case('n_a%d-%s' % (_na, _v), _v, 128, 8, 'n_a != 4: the non-float4 head / dh branches', n_a=_na)
# the edges of the shape envelope (tests/shape_cases.py) on every instantiation and on the fused rollout + BPTT path
for _v in ('ma2c_nc', 'ma2c_ic3'):
    _case('k30-' + _v, _v, 128, 8, 'n_s = 10, K = 30: the last k-step of the encoder k-block is partly padding', n_s=10)
for _v in ('ma2c_nc', 'ia2c'):
    _case('k32-ladder-' + _v, _v, 128, 8, '2x4 ladder, n_s = 8: K = 32 exactly for the inner agents, 24 for the corners',
          topo='ladder8', n_s=8)
_case('k32-ma2c_cu', 'ma2c_cu', 128, 8, 'n_s = 32: a single-source encoder that fills its k-block', n_s=32)
_case('n_a3-ma2c_dial', 'ma2c_dial', 128, 8, 'n_a = 3: the generic heads beside the n_a == 4 fast path', n_a=3)
_case('n_a1-ma2c_nc', 'ma2c_nc', 128, 8, 'n_a = 1: pi == 1, zero logit gradients', n_a=1)
for _v in ('ma2c_nc', 'ia2c'):
    _case('wgrad-kb20-' + _v, _v, 128, 160, '20 k-blocks per split: one full segment, idle last split', kb=(20, [20]))
    _case('wgrad-kb21-' + _v, _v, 128, 168, '21 k-blocks per split: a 20-block segment then a 1-block segment',
          kb=(21, [20, 1]))
    _case('wgrad-kb41-' + _v, _v, 256, 166, '41 k-blocks per split: 20 + 20 + 1, partial last split', kb=(41, [20, 20, 1]))


# ---- float64 round-off scale of every parameter entry -------------------------------------------------------------
class RoundoffScale(TorchFunctionMode):
    """Active around the oracle's forward + backward: every x @ W and every (.. + b) with a leaf parameter W / b hooks
    the gradient delta of its output and accumulates S_W += |x|^T |delta|, S_b += sum over rows |delta|.  The hooks
    only read; the oracle's numbers are unchanged.

    It also collects K, the part of each gradient entry that hinges on a ReLU kink: where an encoder pre-activation z
    of W / b lies within KINK of 0, an fp32 kernel computes z with the opposite sign as legitimately as not (the fp32
    error of z is ~1e-6), and the row's gradient then passes the ReLU or not.  K_W = |x|^T |delta_z| and K_b = |delta_z|
    summed over those rows bound that difference."""
    MATMUL = {torch.matmul, torch.Tensor.matmul, torch.Tensor.__matmul__}
    ADD = {torch.add, torch.Tensor.add, torch.Tensor.__add__, torch.Tensor.__radd__}
    RELU = {torch.relu, torch.Tensor.relu, torch.nn.functional.relu}

    def __init__(self, params):
        super().__init__()
        self.name = {id(t): n for n, t in params.items()}
        self.S = {n: torch.zeros_like(t, requires_grad=False) for n, t in params.items()}
        self.K = {n: torch.zeros_like(t, requires_grad=False) for n, t in params.items()}
        self.keep = []                 # the tensors the maps below are keyed by (ids stay unique while they live)
        self.sum_of = {}               # id(x @ W) -> id(x @ W + b)
        self.kink = {}                 # id(z) -> |gradient of relu(z)| on the rows where |z| < KINK, set in backward

    def __exit__(self, *exc):
        # the hooks hold this object, and the tensors in `keep` hold the hooks inside autograd's C++ graph: a cycle the
        # Python collector cannot see, which would keep every hooked activation (and x) alive for good.  The backward
        # has run inside the mode, so drop the tensors; S and K stay.
        self.keep.clear(); self.sum_of.clear(); self.kink.clear()
        return super().__exit__(*exc)

    def _acc(self, d, n, val):
        with torch.no_grad():
            d[n] += val

    def _rows(self, t):
        return t.reshape(int(np.prod(t.shape[:-1])), t.shape[-1])     # also [B, 0]: an empty neighbour input

    def __torch_function__(self, func, types, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        if not (isinstance(out, torch.Tensor) and out.requires_grad):
            return out
        if func in self.MATMUL and id(args[1]) in self.name:
            n, x = self.name[id(args[1])], args[0].detach().abs()
            key = id(out)

            def hook(g, n=n, x=x, key=key):
                self._acc(self.S, n, self._rows(x).T @ self._rows(g.abs()))
                amb = self.kink.get(self.sum_of.get(key))
                if amb is not None:
                    self._acc(self.K, n, self._rows(x).T @ self._rows(amb))
            out.register_hook(hook)
            self.keep.append(out)
        elif func in self.ADD:
            for a, other in ((args[0], args[1]), (args[1], args[0])):
                if isinstance(a, torch.Tensor) and id(a) in self.name:
                    n, key = self.name[id(a)], id(out)
                    self.sum_of[id(other)] = key

                    def hook(g, n=n, key=key):
                        self._acc(self.S, n, self._rows(g.abs()).sum(0))
                        amb = self.kink.get(key)
                        if amb is not None:
                            self._acc(self.K, n, self._rows(amb).sum(0))
                    out.register_hook(hook)
                    self.keep.append(out)
        elif func in self.RELU:
            z = args[0]
            near = (z.detach().abs() < KINK).to(z.dtype)
            if near.any():
                out.register_hook(lambda g, key=id(z), near=near: self.kink.__setitem__(key, g.abs() * near))
                self.keep.append(z)
        return out


# ---- set-up ----------------------------------------------------------------------------------------------------------
def _model(c):
    from deeprl_network_b200.envs.cacc_env import grid_masks
    from deeprl_network_b200.layout import HeteroLayout, ModelLayout
    v = c['variant']
    if c['topo'].startswith('hetero'):
        g = golden(c['topo'] + '_' + v)
        n_s, n_a, mask = [int(x) for x in g['n_s_ls']], [int(x) for x in g['n_a_ls']], g['mask']
        lay = HeteroLayout(v, n_s, n_a, mask)
        return lay, (v, n_s, n_a, mask), n_s, n_a
    if c['topo'] == 'ladder8':
        mask = ladder_masks(4)
    else:
        mask = grid_masks(5)[0] if c['topo'] == 'grid5' else chain_masks(32 if c['topo'] == 'chain32' else 8)[0]
    if c['topo'] == 'chain8cut':
        mask[CUT, :] = 0; mask[:, CUT] = 0
    N, n_a = len(mask), c['n_a']
    n_s_ls = widths(v, mask, c['n_s'], n_a)
    lay = ModelLayout(v, n_s_ls, n_a, mask, obs_mode='gather')
    return lay, (v, n_s_ls, n_a, mask), [c['n_s']] * N, [n_a] * N


def _done_pattern(kind, rs, T, B):
    d = np.zeros((T + 1, B), dtype=np.float32)
    if kind == 't0':
        d[0] = 1
    elif kind == 'block':
        d[0, ::2] = 1; d[3, 32:64] = 1
    elif kind == 'cta':
        d[2, 63] = 1; d[2, 64] = 1; d[5, 127:129] = 1
    elif kind == 'all':
        d[4] = 1
    else:                               # half the envs start fresh, then sparse episode ends (and a bootstrap done)
        d[0, ::2] = 1
        d[1:] = rs.rand(T, B) < 0.03
    return d


def _inputs(c, n_s, n_a, seed=0):
    rs = np.random.RandomState(seed)
    T, B, N = c['T'], c['B'], len(n_s)
    W = max(n_s)

    def fps(shape):
        f = np.zeros((*shape, N, max(n_a)), dtype=np.float32)
        for i in range(N):
            f[..., i, :n_a[i]] = rs.dirichlet(np.ones(n_a[i]), size=shape)
        return f
    base = rs.randn(T + 1, B, N, W).astype(np.float32)
    for i in range(N):
        base[..., i, n_s[i]:] = 0
    x = dict(base=base, fp=fps((T, B)), fp0=fps((B,)),
             acts=np.stack([rs.randint(0, n_a[i], size=(T, B)) for i in range(N)], axis=-1),
             dones=_done_pattern(c['dones'], rs, T, B),
             Rs=rs.randn(T, B, N).astype(np.float32), Advs=rs.randn(T, B, N).astype(np.float32),
             c0=(rs.randn(B, N, NH) * .5).astype(np.float32), h0=(np.tanh(rs.randn(B, N, NH)) * .8).astype(np.float32),
             uni=rs.rand(T + 1, N, B))
    x['fp'][0] = x['fp0']
    return x


def _engine(lay, params, c, tc):
    from deeprl_network_b200.agents.engine import PolicyEngine
    e = PolicyEngine(lay, c['B'], c['T'], dict(HP), flat_params=lay.pack(params), use_tc=tc)
    assert e.use_tc == tc, 'the shape must select the path under test'
    assert e.state_fm == (tc and e.variant != 'ma2c_dial'), 'feature-major state on the tensor-core path, but DIAL'
    return e


def _kernel_advs(lay, Advs):
    # heterogeneous layouts: the kernels get the advantages summed over agents (engine.compute_returns, quirk Q7)
    return np.repeat(Advs.sum(-1, keepdims=True), Advs.shape[-1], -1) if getattr(lay, 'hetero', False) else Advs


def _states(e, t0, t1):
    """h_seq / c_seq slots [t0, t1) -> env-major [t, B, N, 64]"""
    out = []
    for s in (e.c_seq, e.h_seq):
        x = s[t0:t1]
        x = x.permute(0, 3, 1, 2) if e.state_fm else x.permute(0, 2, 1, 3)
        out.append(x.cpu().numpy())
    return out


def _result(e, lay):
    torch.cuda.synchronize()
    e.check_tc()
    flat = e.grads.cpu().numpy()
    return dict(flat=flat, g=lay.unpack(flat), losses=e.losses())


def _run_unfused(e, lay, x, fp, acts, W):
    T = e.T
    e.T_cur = T
    e.obs_buf.zero_()
    e.obs_buf[:T, :, :, :W].copy_(to_dev(np.transpose(x['base'][:T], (0, 2, 1, 3))))
    e.fp_buf[:T].copy_(to_dev(np.transpose(fp, (0, 2, 1, 3))))
    e.act_buf[:T].copy_(to_dev(np.transpose(acts, (0, 2, 1)), torch.int32))
    e.done_buf[:T].copy_(to_dev(x['dones'][:T]))
    e.Rs[:T].copy_(to_dev(np.transpose(x['Rs'], (0, 2, 1))))
    e.Advs[:T].copy_(to_dev(np.transpose(_kernel_advs(lay, x['Advs']), (0, 2, 1))))
    e.set_states(nb(x['c0']), nb(x['h0']))
    e.backward()
    r = _result(e, lay)
    r['c'], r['h'] = _states(e, 1, T + 1)
    return r


def _run_fused(e, lay, x, W):
    T, N, B = e.T, e.N, e.B
    obs = torch.zeros(T + 1, N, B, lay.obs_stride, device='cuda')
    obs[..., :W] = to_dev(np.transpose(x['base'], (0, 2, 1, 3)))
    dones = to_dev(x['dones'])
    e.obs_buf[0].copy_(obs[0]); e.fp_buf[0].copy_(nb(x['fp0'])); e.done_buf[0].copy_(dones[0])
    e.set_states(nb(x['c0']), nb(x['h0']))
    e.rollout(ScriptedEnv(obs, dones), sample='uniform', uniforms=to_dev(x['uni'], torch.float64))
    assert e.saved_rollout, 'the fused path (rollout p-calls save the BPTT activations) must be the one under test'
    torch.cuda.synchronize()
    rec = dict(fp=np.transpose(e.fp_buf.cpu().numpy(), (0, 2, 1, 3)), acts=np.transpose(e.act_buf.cpu().numpy(), (0, 2, 1)),
               v=np.transpose(e.val_buf.cpu().numpy(), (0, 2, 1)))
    np.testing.assert_array_equal(e.done_buf.cpu().numpy(), x['dones'])
    c, h = _states(e, 1, T + 1)
    # the rollout's Rs / Advs come from zero rewards; the test's own values make the policy loss non-trivial
    e.Rs[:T].copy_(to_dev(np.transpose(x['Rs'], (0, 2, 1))))
    e.Advs[:T].copy_(to_dev(np.transpose(_kernel_advs(lay, x['Advs']), (0, 2, 1))))
    e.backward()
    r = _result(e, lay)
    r.update(rec, c=c, h=h)
    return r


def _oracle(lay, orc_args, params, c, x, n_s, fp, acts):
    T, B, N = c['T'], c['B'], len(n_s)
    orc = nets.OraclePolicy(*orc_args, params=params, dtype=torch.float64, n_env=B)
    if c['topo'].startswith('hetero'):
        obs = [[x['base'][t][:, i, :n_s[i]] for i in range(N)] for t in range(T)]
    else:
        obs = [oracle_obs(lay, x['base'][t]) for t in range(T)]
    st = torch.tensor(np.concatenate([x['c0'], x['h0']], -1), dtype=torch.float64)
    orc.states_bw = st.clone()
    mode = RoundoffScale(orc.p)
    with mode:
        summ = orc.backward(obs, fp.astype(np.float64), acts, x['dones'][:T], x['Rs'], x['Advs'], 5e-4,
                            v_coef=HP['v_coef'], e_coef=HP['e_coef'], apply=False)
    cs, hs, vs = [], [], []
    with torch.no_grad():                  # the states the training forward went through
        cc, hh = st[..., :NH], st[..., NH:]
        for t in range(T):
            xt, pt = orc._prep(obs[t], fp[t].astype(np.float64))
            d = torch.as_tensor(x['dones'][t], dtype=torch.float64)
            cc, hh = orc._cell(xt, pt, d, cc, hh)
            cs.append(cc.numpy()); hs.append(hh.numpy())
            # the rollout's v-call re-runs the cell from the state the p-call just stored (quirk Q1), so its v is
            # not the training forward's v
            _, h2 = orc._cell(xt, pt, d, cc, hh)
            a = torch.as_tensor(np.asarray(acts[t]), dtype=torch.int64)
            vs.append(torch.stack([orc._v(i, h2[:, i], a) for i in range(N)], dim=1).numpy())
    return dict(g={n: orc.grads[n].numpy() for n in orc.names}, S={n: mode.S[n].numpy() for n in orc.names},
                K={n: mode.K[n].numpy() for n in orc.names},
                summ=summ, pi=orc.last_pi.numpy(), v_roll=np.stack(vs), c=np.stack(cs), h=np.stack(hs))


def _used(lay):
    used = np.zeros(lay.n_param, bool)
    if getattr(lay, 'hetero', False):
        for n in lay._idx:
            used[lay._idx[n]] = True
    else:
        for _, o, s in lay.entries:
            used[o:o + int(np.prod(s))] = True
    return used


def _check(tag, r, ref, used):
    """per-tensor checks of one run against the oracle; returns {tensor: per-entry ratio max|g - g64| / S}"""
    ratios = {}
    for n, g64 in ref['g'].items():
        if g64.size == 0:              # the [0, 64] fingerprint / message weights of an agent without neighbours
            continue
        err = np.maximum(np.abs(r['g'][n] - g64) - ref['K'][n], 0)        # minus what a ReLU kink may flip
        scale = max(1e-3, np.abs(g64).max())
        assert err.max() <= 2e-5 * scale + 1e-7, (tag, n, err.max(), scale)
        ratios[n] = float((err / np.maximum(ref['S'][n], S_REL * ref['S'][n].max() + 1e-300)).max())
    s = ref['summ']
    for k in ('policy_loss', 'value_loss', 'entropy_loss'):
        np.testing.assert_allclose(r['losses'][k], s[k], rtol=1e-4, atol=1e-5, err_msg='%s %s' % (tag, k))
    assert np.all(r['flat'][~used] == 0), (tag, 'the layout padding must receive exactly zero gradient')
    for k in ('c', 'h'):
        err = np.abs(r[k] - ref[k]).max()
        assert err < 1e-5, (tag, 'state ' + k, err)
    if 'v' in r:
        assert np.abs(r['fp'][1:] - ref['pi']).max() < 1e-5, (tag, 'pi', np.abs(r['fp'][1:] - ref['pi']).max())
        assert np.abs(r['v'] - ref['v_roll']).max() < 1e-5, (tag, 'v', np.abs(r['v'] - ref['v_roll']).max())
    return ratios


@pytest.mark.parametrize('mode', ['unfused', 'fused'])
@pytest.mark.parametrize('c', CASES)
def test_tc_paths_match_fp64(c, mode):
    lay, orc_args, n_s, n_a = _model(c)
    B, T, N = c['B'], c['T'], lay.N
    if c['kb'] is not None:            # the weight-gradient regime the case is named after
        per, last = wgrad_kb_per_split(B, T, N)
        assert per == c['kb'][0] and last < per
        assert [min(SEG_KB, per - s) for s in range(0, per, SEG_KB)] == c['kb'][1]
    if c['topo'] == 'chain32':
        assert wgrad_splits(N) == 5
    if c['topo'] in ('hetero_iso', 'chain8cut'):
        assert [i for i in range(N) if lay.nbr[i] == []] == [N - 1 if c['topo'] == 'hetero_iso' else CUT]
    if c['topo'] == 'grid5':
        assert wgrad_splits(N) == 9 and sorted({int(k) for k in orc_args[3].sum(1)}) == [2, 3, 4]
    params = random_params(lay.creation_order(), seed=3, scale=0.3)
    x = _inputs(c, n_s, n_a)
    W = max(n_s)
    used = _used(lay)
    e = _engine(lay, params, c, tc=True)
    r = _run_unfused(e, lay, x, x['fp'], x['acts'], W) if mode == 'unfused' else _run_fused(e, lay, x, W)
    del e
    fp, acts = (x['fp'], x['acts']) if mode == 'unfused' else (r['fp'][:T], r['acts'])
    ref = _oracle(lay, orc_args, params, c, x, n_s, fp, acts)
    # calibration: the FP32-FFMA kernels on the same buffers against the same oracle
    e = _engine(lay, params, c, tc=False)
    ffma = _run_unfused(e, lay, x, fp, acts, W)
    del e
    r_ffma = _check('%s ffma' % mode, ffma, ref, used)
    tag = '%s tc' % mode
    r_tc = _check(tag, r, ref, used)
    bad = {n: (r_tc[n], r_ffma[n]) for n in r_tc if r_tc[n] > 4 * r_ffma[n] + FLOOR}
    assert not bad, (tag, 'per-entry error / round-off scale', sorted(bad.items(), key=lambda t: -t[1][0])[:6])
    print('[%s] %s B=%d T=%d N=%d worst per-entry ratio: tc %.2e ffma %.2e' % (
        c['purpose'], mode, B, T, N, max(r_tc.values()), max(r_ffma.values())))
