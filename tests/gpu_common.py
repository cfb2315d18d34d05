"""Helpers shared by the GPU parity tests: build a CUDA engine and an oracle policy holding the
same weights, and convert between the kernel layout [agent][env][..] and the oracle's [env][agent][..]."""
import numpy as np
import torch

from helpers import random_params
from oracle import nets
from oracle.cacc import chain_masks

N_S = {'ia2c': [10, 15, 15, 15, 15, 15, 15, 10]}
HP = dict(v_coef=0.5, e_coef=0.05, max_grad_norm=40.0, alpha=0.99, epsilon=1e-5, gamma=0.99,
          reward_norm=5000.0, reward_clip=-1.0)


def ladder_masks(cols=4):
    """2 x cols ladder, row-major: the corner agents have 2 neighbours, the inner ones 3."""
    r, c = np.divmod(np.arange(2 * cols), cols)
    return ((np.abs(r[:, None] - r[None, :]) + np.abs(c[:, None] - c[None, :])) == 1).astype(int)


def cut_chain_mask(n=8, cut=3):
    """n-agent chain with agent `cut` cut off: it has no neighbours, and is nobody's neighbour."""
    mask = chain_masks(n)[0]
    mask[cut, :] = 0; mask[:, cut] = 0
    return mask


def widths(variant, mask, n_s, n_a):
    """n_s_ls as the agents classes count it for an own-observation width n_s (gathered observations)."""
    nm = [int(np.asarray(mask)[i].sum()) for i in range(len(mask))]
    return {'ia2c': [n_s * (1 + k) for k in nm],
            'ia2c_fp': [n_s * (1 + k) + n_a * k for k in nm]}.get(variant, [n_s] * len(mask))


def make_pair(variant, B, T=4, seed=0, dtype=torch.float32, mask=None, n_a=4, hp=None, scale=0.3, n_s=5):
    from deeprl_network_b200.agents.engine import PolicyEngine
    from deeprl_network_b200.layout import ModelLayout
    if mask is None:
        mask, _ = chain_masks(8)
    N = len(mask)
    n_s_ls = widths(variant, mask, n_s, n_a)
    lay = ModelLayout(variant, n_s_ls, n_a, mask, obs_mode='gather')
    params = random_params(lay.creation_order(), seed=seed, scale=scale)
    eng = PolicyEngine(lay, B, T, dict(HP if hp is None else hp), flat_params=lay.pack(params))
    orc = nets.OraclePolicy(variant, n_s_ls, n_a, mask, params=params, dtype=dtype, n_env=B)
    return eng, orc, lay, params


def check_apply_twice(eng, orc, lay, pad, lr=1e-2):
    """Two clip + RMSProp steps on the gradients of the last backward (the second one with ms != 1): norm_out equals
    the oracle's global norm(s), the weights follow the oracle's, and every padding float (`pad`) stays exactly 0."""
    for _ in range(2):
        eng.apply(lr)
        norms = orc.apply_grads(lr, max_grad_norm=HP['max_grad_norm'], alpha=HP['alpha'], epsilon=HP['epsilon'])
        torch.cuda.synchronize()
        np.testing.assert_allclose(eng.norm_out.cpu().numpy(), norms, rtol=1e-4)
        flat = eng.params.cpu().numpy()
        assert np.all(flat[pad] == 0), 'padding moved'
        w = lay.unpack(flat)
        for n in orc.names:
            np.testing.assert_allclose(w[n], orc.p[n].detach().numpy(), rtol=0, atol=3e-6, err_msg=n)


def oracle_obs(lay, base):
    """base [B, N, n_s] own features -> per-agent oracle inputs (IA2C: own + neighbours concatenated; pre-concatenated
    observations of unequal width: the agent's first n_s_ls[i] columns)."""
    if lay.concat:
        return [base[:, i, :lay.n_s_ls[i]] for i in range(lay.N)]
    if lay.variant not in ('ia2c', 'ia2c_fp'):      # ia2c_fp: the fingerprints travel separately (ps)
        return [base[:, i] for i in range(lay.N)]
    return [np.concatenate([base[:, i]] + [base[:, j] for j in lay.nbr[i]], axis=1) for i in range(lay.N)]


def to_dev(x, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).cuda()


def nb(x):
    """[B, N, ...] -> contiguous [N, B, ...] device tensor."""
    return to_dev(np.swapaxes(x, 0, 1))


def bn(t):
    """device [N, B, ...] -> numpy [B, N, ...]."""
    return np.swapaxes(t.detach().cpu().numpy(), 0, 1)


def obs_dev(lay, base, poison=False):
    """base [B, N, w] -> device observation rows [N, B, obs_stride].  Agent i owns its first w columns (n_s_ls[i] of
    them when the rows are pre-concatenated observations of unequal width); the columns behind them are padding, which
    the kernels never read: zero, or NaN with `poison`."""
    B, N, w = base.shape
    o = np.full((N, B, lay.obs_stride), np.nan if poison else 0.0, dtype=np.float32)
    for i in range(N):
        wi = lay.n_s_ls[i] if lay.concat else w
        o[i, :, :wi] = base[:, i, :wi]
    return to_dev(o)


class ScriptedEnv:
    """Device stand-in for CACCEnv in `PolicyEngine.rollout`: step t writes the pre-generated observations and dones of
    slot t + 1 (and zero rewards), whatever actions were sampled.  Lets the fused rollout path (rollout p-calls that
    save the BPTT activations, then `backward`) run on any layout -- heterogeneous ones included -- and any done
    pattern.  obs: device [T+1, N, B, obs_stride]; done: device [T+1, B] (slot t = done before step t)."""

    def __init__(self, obs, done):
        self.obs, self.done, self.t = obs, done, 0

    def step_device(self, action, obs_out=None, reward_out=None, greward_out=None, done_out=None):
        self.t += 1
        obs_out.copy_(self.obs[self.t])
        done_out.copy_(self.done[self.t])
        reward_out.zero_()
        greward_out.zero_()
