"""CPU oracle for heterogeneous IA2C / IA2C_FP / IA2C_CU agents (the reference's ``identical_agent == False`` path
of LstmPolicy, FPPolicy and ConsensusPolicy), restated in PyTorch-CPU on top of ``oracle.nets.OraclePolicy``.

  * IA2C     ``LstmPolicy(n_s_ls[i], n_a_ls[i], ..., na_dim_ls, identical=False)``  agents/models.py:118-132
             fc on the agent's own observation; pi head n_a_i wide; the value head concatenates h with one one-hot
             per neighbour j of width n_a_j (``_build_critic_head``, agents/policies.py:59-77)
  * IA2C_FP  ``FPPolicy``  agents/models.py:171-188, agents/policies.py:157-185: the observation is the agent's own
             n_s_ls[i] features followed by the neighbours' policies (n_a_j each); fcs takes the former, fcp the
             latter; without neighbours there is no fcp and lstm/wx is [n_fc, 4 n_h]
  * IA2C_CU  ``ConsensusPolicy``  agents/models.py:261-275, agents/policies.py:366-426: observations zero-padded
             to max(n_s_ls) (agents/models.py:229-235), fc_%da on the padded width, actor head cu/pi_%da, the
             non-identical prepare_loss branch (quirk Q7, agents/policies.py:241-251) and the consensus update

Pinned to the unmodified reference on the TF shim by tests/golden/hetero_{,iso_,iso0_}{ia2c,ia2c_fp,ma2c_cu}.npz
(tests/test_hetero_ia2c_parity.py).
"""
import numpy as np
import torch

from oracle import nets

VARIANTS = ('ia2c', 'ia2c_fp', 'ma2c_cu')


def param_shapes(variant, n_s_ls, n_a_ls, mask, n_h=64, n_fc=64):
    """(name, shape) in tf.get_variable order: one policy after the other, heads last within each.  n_s_ls are the
    agents' own observation widths (IA2C_FP: without the fingerprints)."""
    N = len(mask)
    nbr = [list(np.where(np.asarray(mask)[i] == 1)[0]) for i in range(N)]
    out = []
    for i in range(N):
        kp = sum(n_a_ls[j] for j in nbr[i])
        if variant == 'ma2c_cu':
            s, pi, v = 'cu/fc_%da' % i, 'cu/pi_%da' % i, 'cu/v_%da' % i
            out += [(s + '/w', (max(n_s_ls), n_h)), (s + '/b', (n_h,))]
            lstm = 'cu/lstm_%da' % i
            n_in = n_h
        else:
            s = 'lstm_%d' % i
            pi, v, lstm = s + '/pi', s + '/v', s + '/lstm'
            if variant == 'ia2c':
                out += [(s + '/fc/w', (n_s_ls[i], n_fc)), (s + '/fc/b', (n_fc,))]
                n_in = n_fc
            else:
                out += [(s + '/fcs/w', (n_s_ls[i], n_fc)), (s + '/fcs/b', (n_fc,))]
                if nbr[i]:
                    out += [(s + '/fcp/w', (kp, n_fc)), (s + '/fcp/b', (n_fc,))]
                n_in = 2 * n_fc if nbr[i] else n_fc
        out += [(lstm + '/wx', (n_in, 4 * n_h)), (lstm + '/wh', (n_h, 4 * n_h)), (lstm + '/b', (4 * n_h,)),
                (pi + '/w', (n_h, n_a_ls[i])), (pi + '/b', (n_a_ls[i],)), (v + '/w', (n_h + kp, 1)), (v + '/b', (1,))]
    return out


class HeteroIA2COracle(nets.OraclePolicy):
    """``OraclePolicy`` for heterogeneous IA2C / IA2C_FP / IA2C_CU.  Same protocol: ``forward`` takes per-agent
    observations ([B, n_s_i]; IA2C_FP either with the fingerprints appended or without them plus ``ps``) and
    returns per-agent policies of tight width; ``backward`` / ``apply_grads`` / ``consensus_update`` as there."""

    def __init__(self, variant, n_s_ls, n_a_ls, mask, n_h=64, n_fc=64, params=None, dtype=torch.float32, n_env=1):
        assert variant in VARIANTS and nets.is_hetero(n_a_ls)
        self.hetero = True
        self.n_a_ls = [int(a) for a in n_a_ls]
        self.variant, self.n_a, self.n_h, self.n_fc = variant, max(self.n_a_ls), n_h, n_fc
        self.mask = np.asarray(mask)
        self.N = len(self.mask)
        self.nbr = [list(np.where(self.mask[i] == 1)[0]) for i in range(self.N)]
        self.n_s_ls = [int(x) for x in n_s_ls]
        self.dtype, self.B = dtype, n_env
        shapes = param_shapes(variant, self.n_s_ls, self.n_a_ls, mask, n_h, n_fc)
        if params is None:
            params = {n: nets.ortho_init(s) if len(s) == 2 else np.zeros(s, dtype=np.float32) for n, s in shapes}
        self.names = [n for n, _ in shapes]
        self.p = {n: torch.tensor(np.asarray(params[n]), dtype=dtype).requires_grad_(True) for n in self.names}
        self.ms = {n: torch.ones_like(self.p[n]) for n in self.names}
        self.reset()

    def _head(self, i, key):
        if self.variant == 'ma2c_cu':
            a, b = key.split('/')
            return self.p['cu/%s_%da/%s' % (a, i, b)]
        return super()._head(i, key)

    def _prep(self, obs, ps):
        x, p = super()._prep(obs, ps)
        if self.variant == 'ma2c_cu':       # MA2C_NC._convert_hetero_states: zero-pad to max(n_s_ls)
            ns = max(self.n_s_ls)
            x = [torch.cat([xi, torch.zeros(xi.shape[0], ns - xi.shape[1], dtype=self.dtype)], dim=1) for xi in x]
        return x, p

    def _cell(self, x, p, done, c, h):
        if self.variant != 'ia2c_fp':
            return super()._cell(x, p, done, c, h)
        nd = (1.0 - done).unsqueeze(-1)
        new_c, new_h = [], []
        for i in range(self.N):
            ci, hi = c[:, i] * nd, h[:, i] * nd
            nb, n_x = self.nbr[i], self.n_s_ls[i]
            s = torch.relu(x[i][:, :n_x] @ self._w(i, 'fcs/w') + self._w(i, 'fcs/b'))
            if nb:
                # fingerprints inside the observation, or (batched tests) from `p` with each neighbour's n_a_j entries
                fp_in = x[i][:, n_x:] if x[i].shape[1] > n_x else torch.cat([p[:, j, :self.n_a_ls[j]] for j in nb], dim=1)
                s = torch.cat([s, torch.relu(fp_in @ self._w(i, 'fcp/w') + self._w(i, 'fcp/b'))], dim=1)
            z = s @ self._w(i, 'lstm/wx') + hi @ self._w(i, 'lstm/wh') + self._w(i, 'lstm/b')
            ig, fg, og, ug = torch.split(z, self.n_h, dim=1)
            ci = torch.sigmoid(fg) * ci + torch.sigmoid(ig) * torch.tanh(ug)
            hi = torch.sigmoid(og) * torch.tanh(ci)
            new_c.append(ci); new_h.append(hi)
        return torch.stack(new_c, dim=1), torch.stack(new_h, dim=1)

    def loss_terms(self, pi, v, acts, Rs, Advs, v_coef, e_coef):
        if self.variant == 'ma2c_cu':       # NCMultiAgentPolicy.prepare_loss, non-identical branch: quirk Q7
            return super().loss_terms(pi, v, acts, Rs, Advs, v_coef, e_coef)
        # IA2C / IA2C_FP: one Policy.prepare_loss per agent (agents/policies.py:20-30), no broadcast across agents
        a = torch.as_tensor(np.asarray(acts), dtype=torch.int64)
        R = torch.as_tensor(np.asarray(Rs), dtype=self.dtype)
        A = torch.as_tensor(np.asarray(Advs), dtype=self.dtype)
        log_pi = torch.log(torch.clamp(pi, 1e-10, 1.0))
        ent = -(pi * log_pi).sum(-1)
        lp = torch.gather(log_pi, -1, a.unsqueeze(-1)).squeeze(-1)
        return -(lp * A).mean(dim=(0, 1)), ((R - v) ** 2).mean(dim=(0, 1)) * 0.5 * v_coef, -ent.mean(dim=(0, 1)) * e_coef
