"""CPU oracle: the TF1 policy graphs, A2C loss, global-norm clip and TF-RMSProp,
restated in PyTorch-CPU (fp32 by default, fp64 switch).

TEST INFRASTRUCTURE -- see ``oracle/__init__.py``.
PINNED to the reference's own network source executed on a TF shim (tests/golden/tf_shim.py,
tests/test_tfnet_parity.py: pi / v / R within 2e-7 and trained weights within 3e-8 of the unmodified
reference code for all six agents); TensorFlow 1.12 (README.md:23) itself cannot be installed here, so the
TF primitives' own semantics (incl. the clip / RMSProp formulas below) remain restated, not measured.
This file is a line-by-line restatement of

  * ``fc``            agents/utils.py:65-73        * ``ortho_init``  agents/utils.py:10-23
  * ``lstm``          agents/utils.py:87-115       (IA2C / LstmPolicy, policies.py:136-149)
  * ``lstm_comm``     agents/utils.py:118-217      (NeurComm)
  * ``lstm_ic3``      agents/utils.py:344-417      (CommNet)
  * ``lstm_dial``     agents/utils.py:515-599      (DIAL)
  * ``lstm_comm_hetero`` / ``lstm_ic3_hetero`` / ``lstm_dial_hetero``  agents/utils.py:220-341, 420-512, 602-702
    (agents with unequal observation / action widths: pass ``n_a`` as a list; pinned by tests/golden/hetero_*.npz,
    which ran the unmodified reference classes on the TF shim)
  * heads             agents/policies.py:50-77, 291-312
  * loss              agents/policies.py:20-39 (IA2C, per agent) / :232-264 (MA2C)
  * stateful forward/backward protocol  agents/policies.py:103-134, 200-230, 334-336
  * TF numerics (SURVEY a23): clip_by_global_norm g*clip/max(|g|,clip);
    RMSProp ms0=1, ms=rho*ms+(1-rho)g^2, w-=lr*g/sqrt(ms+eps) (eps INSIDE the sqrt)

Extension over the reference: a leading env axis B.  B=1 is exactly the reference;
for B>1 ``mean_t`` in the loss becomes the mean over (b,t) (SURVEY A.4).
Gate order is i,f,o,u; state layout is [c | h].
"""
import numpy as np
import torch

VARIANTS = ('ia2c', 'ia2c_fp', 'ma2c_cu', 'ma2c_nc', 'ma2c_ic3', 'ma2c_dial')
SCOPE = {'ma2c_nc': 'nc', 'ma2c_ic3': 'ic3', 'ma2c_dial': 'dial'}
CELL = {'ma2c_nc': 'lstm_comm', 'ma2c_ic3': 'lstm_ic3', 'ma2c_dial': 'lstm_comm'}


def ortho_init(shape, scale=np.sqrt(2)):
    """agents/utils.py:10-23 -- consumes the GLOBAL numpy stream."""
    a = np.random.standard_normal(shape)
    u, _, v = np.linalg.svd(a, full_matrices=False)
    q = u if u.shape == tuple(shape) else v
    return (scale * q.reshape(shape)).astype(np.float32)


def is_hetero(n_a):
    """n_a given per agent with unequal entries (agents/models.py:89-97: identical_agent iff all n_a equal)."""
    return (not np.isscalar(n_a)) and len(set(int(a) for a in n_a)) > 1


def param_shapes(variant, n_s_ls, n_a, mask, n_h=64, n_fc=64):
    """Ordered (name, shape, is_weight) list in the reference's tf.get_variable order
    (SURVEY A.5); biases are interleaved where the reference creates them."""
    N = len(mask)
    nm = [int(np.sum(mask[i])) for i in range(N)]
    out = []
    if variant == 'ia2c':
        for i in range(N):
            s = 'lstm_%d' % i
            out += [(s + '/fc/w', (n_s_ls[i], n_fc)), (s + '/fc/b', (n_fc,)),
                    (s + '/lstm/wx', (n_fc, 4 * n_h)), (s + '/lstm/wh', (n_h, 4 * n_h)), (s + '/lstm/b', (4 * n_h,)),
                    (s + '/pi/w', (n_h, n_a)), (s + '/pi/b', (n_a,)),
                    (s + '/v/w', (n_h + n_a * nm[i], 1)), (s + '/v/b', (1,))]
        return out
    if variant == 'ia2c_fp':     # FPPolicy (agents/policies.py:157-185); n_s_ls already counts the fingerprints
        for i in range(N):
            s = 'lstm_%d' % i
            n_x = n_s_ls[i] - n_a * nm[i]
            out += [(s + '/fcs/w', (n_x, n_fc)), (s + '/fcs/b', (n_fc,)),
                    (s + '/fcp/w', (n_a * nm[i], n_fc)), (s + '/fcp/b', (n_fc,)),
                    (s + '/lstm/wx', (2 * n_fc, 4 * n_h)), (s + '/lstm/wh', (n_h, 4 * n_h)), (s + '/lstm/b', (4 * n_h,)),
                    (s + '/pi/w', (n_h, n_a)), (s + '/pi/b', (n_a,)),
                    (s + '/v/w', (n_h + n_a * nm[i], 1)), (s + '/v/b', (1,))]
        return out
    if variant == 'ma2c_cu':     # ConsensusPolicy._build_net (agents/policies.py:366-399)
        for i in range(N):
            out += [('cu/fc_%da/w' % i, (n_s_ls[i], n_h)), ('cu/fc_%da/b' % i, (n_h,)),
                    ('cu/lstm_%da/wx' % i, (n_h, 4 * n_h)), ('cu/lstm_%da/wh' % i, (n_h, 4 * n_h)), ('cu/lstm_%da/b' % i, (4 * n_h,)),
                    ('cu/pi_%d/w' % i, (n_h, n_a)), ('cu/pi_%d/b' % i, (n_a,)),
                    ('cu/v_%da/w' % i, (n_h + n_a * nm[i], 1)), ('cu/v_%da/b' % i, (1,))]
        return out
    sc, cell = SCOPE[variant], CELL[variant]
    if is_hetero(n_a):
        # lstm_*_hetero: tight per-agent widths; NeurComm creates w_ob FIRST here (agents/utils.py:260-283), agents
        # without neighbours have no message / fingerprint encoder and a [n_h, 4 n_h] wx_hid
        n_a_ls = [int(a) for a in n_a]
        nbr = [list(np.where(np.asarray(mask)[i] == 1)[0]) for i in range(N)]
        for i in range(N):
            s = '%s/%s_%d' % (sc, cell, i)
            kx = n_s_ls[i] + sum(n_s_ls[j] for j in nbr[i])
            kp = sum(n_a_ls[j] for j in nbr[i])
            if variant == 'ma2c_nc':
                out += [(s + '/w_ob', (kx, n_h)), (s + '/b_ob', (n_h,))]
                if nm[i]:
                    out += [(s + '/w_fp', (kp, n_h)), (s + '/b_fp', (n_h,)),
                            (s + '/w_msg', (n_h * nm[i], n_h)), (s + '/b_msg', (n_h,))]
                out += [(s + '/wx_hid', ((3 if nm[i] else 1) * n_h, 4 * n_h)), (s + '/wh_hid', (n_h, 4 * n_h)), (s + '/b_hid', (4 * n_h,))]
            else:
                if nm[i]:
                    out += [(s + '/w_msg', (n_h if variant == 'ma2c_ic3' else n_h * nm[i], n_h)), (s + '/b_msg', (n_h,))]
                out += [(s + '/w_ob', (kx, n_h)), (s + '/b_ob', (n_h,)),
                        (s + '/wx_hid', (n_h, 4 * n_h)), (s + '/wh_hid', (n_h, 4 * n_h)), (s + '/b_hid', (4 * n_h,))]
        if variant == 'ma2c_dial':
            for i in range(N):
                out += [('%s/mfc_%d/w' % (sc, i), (n_h, n_h)), ('%s/mfc_%d/b' % (sc, i), (n_h,))]
        for i in range(N):
            out += [('%s/pi_%d/w' % (sc, i), (n_h, n_a_ls[i])), ('%s/pi_%d/b' % (sc, i), (n_a_ls[i],)),
                    ('%s/v_%d/w' % (sc, i), (n_h + sum(n_a_ls[j] for j in nbr[i]), 1)), ('%s/v_%d/b' % (sc, i), (1,))]
        return out
    n_s = n_s_ls[0]
    for i in range(N):
        s = '%s/%s_%d' % (sc, cell, i)
        if variant == 'ma2c_nc':
            out += [(s + '/w_msg', (n_h * nm[i], n_h)), (s + '/b_msg', (n_h,)),
                    (s + '/w_ob', (n_s * (nm[i] + 1), n_h)), (s + '/b_ob', (n_h,)),
                    (s + '/w_fp', (n_a * nm[i], n_h)), (s + '/b_fp', (n_h,)),
                    (s + '/wx_hid', (3 * n_h, 4 * n_h)), (s + '/wh_hid', (n_h, 4 * n_h)), (s + '/b_hid', (4 * n_h,))]
        else:
            km = n_h if variant == 'ma2c_ic3' else n_h * nm[i]
            out += [(s + '/w_msg', (km, n_h)), (s + '/b_msg', (n_h,)),
                    (s + '/w_ob', (n_s * (nm[i] + 1), n_h)), (s + '/b_ob', (n_h,)),
                    (s + '/wx_hid', (n_h, 4 * n_h)), (s + '/wh_hid', (n_h, 4 * n_h)), (s + '/b_hid', (4 * n_h,))]
    if variant == 'ma2c_dial':
        for i in range(N):
            out += [('%s/mfc_%d/w' % (sc, i), (n_h, n_h)), ('%s/mfc_%d/b' % (sc, i), (n_h,))]
    for i in range(N):
        out += [('%s/pi_%d/w' % (sc, i), (n_h, n_a)), ('%s/pi_%d/b' % (sc, i), (n_a,)),
                ('%s/v_%d/w' % (sc, i), (n_h + n_a * nm[i], 1)), ('%s/v_%d/b' % (sc, i), (1,))]
    return out


def init_params(variant, n_s_ls, n_a, mask, n_h=64, n_fc=64):
    """Weights via ortho_init (scale sqrt2, heads included), biases zero.
    Consumes np.random exactly like graph construction does (SURVEY A.5)."""
    p = {}
    for name, shape in param_shapes(variant, n_s_ls, n_a, mask, n_h, n_fc):
        if len(shape) == 2:
            p[name] = ortho_init(shape)
        else:
            p[name] = np.zeros(shape, dtype=np.float32)
    return p


class OraclePolicy:
    """One object per algorithm; holds weights, LSTM states, optimizer slots."""

    def __init__(self, variant, n_s_ls, n_a, mask, n_h=64, n_fc=64, params=None,
                 dtype=torch.float32, n_env=1):
        assert variant in VARIANTS
        self.hetero = is_hetero(n_a)
        if self.hetero:
            assert variant in SCOPE, 'heterogeneous agents exist for ma2c_nc / ma2c_ic3 / ma2c_dial only'
            self.n_a_ls = [int(a) for a in n_a]
            n_a_scalar = max(self.n_a_ls)
        else:
            n_a_scalar = int(n_a if np.isscalar(n_a) else n_a[0])
            self.n_a_ls = [n_a_scalar] * len(mask)
        self._n_a_arg = n_a
        self.variant, self.n_a, self.n_h, self.n_fc = variant, n_a_scalar, n_h, n_fc
        self.mask = np.asarray(mask)
        self.N = len(self.mask)
        self.nbr = [list(np.where(self.mask[i] == 1)[0]) for i in range(self.N)]
        self.n_s_ls = list(n_s_ls)
        self.dtype = dtype
        self.B = n_env
        if params is None:
            params = init_params(variant, n_s_ls, n_a, mask, n_h, n_fc)
        self.names = [n for n, _ in param_shapes(variant, n_s_ls, n_a, mask, n_h, n_fc)]
        self.p = {n: torch.tensor(np.asarray(params[n]), dtype=dtype).requires_grad_(True) for n in self.names}
        self.ms = {n: torch.ones_like(self.p[n]) for n in self.names}   # TF RMSProp slot init = 1
        self.reset()

    # ---- state ---------------------------------------------------------------------
    def reset(self):
        z = torch.zeros(self.B, self.N, 2 * self.n_h, dtype=self.dtype)
        self.states_fw, self.states_bw = z.clone(), z.clone()

    def _w(self, i, key):
        if self.variant in ('ia2c', 'ia2c_fp'):
            return self.p['lstm_%d/%s' % (i, key)]
        if self.variant == 'ma2c_cu':
            a, b = key.split('/')
            return self.p['cu/%s_%da/%s' % (a, i, b)]
        return self.p['%s/%s_%d/%s' % (SCOPE[self.variant], CELL[self.variant], i, key)]

    def _head(self, i, key):
        if self.variant in ('ia2c', 'ia2c_fp'):
            return self.p['lstm_%d/%s' % (i, key)]
        if self.variant == 'ma2c_cu':
            a, b = key.split('/')
            return self.p['cu/%s_%d%s/%s' % (a, i, 'a' if a == 'v' else '', b)]
        sc = SCOPE[self.variant]
        a, b = key.split('/')
        return self.p['%s/%s_%d/%s' % (sc, a, i, b)]

    # ---- one time step of the cell for all agents ------------------------------------
    def _cell(self, x, p, done, c, h):
        """x: list of N [B,n_s_i]; p: [B,N,n_a] or None; done [B]; c,h [B,N,n_h]."""
        nd = (1.0 - done).unsqueeze(-1)
        v = self.variant

        def cat(parts):
            # an agent without neighbours concatenates nothing: a [B, 0] input meets the reference's [0, n_h] weights
            return torch.cat(parts, dim=1) if parts else torch.zeros(c.shape[0], 0, dtype=self.dtype)
        if v == 'ma2c_dial':   # sender-side message fc on the UN-masked h (agents/utils.py:563-566)
            sc = SCOPE[v]
            msg = [torch.relu(h[:, j] @ self.p['%s/mfc_%d/w' % (sc, j)] + self.p['%s/mfc_%d/b' % (sc, j)])
                   for j in range(self.N)]
        new_c, new_h = [], []
        for i in range(self.N):
            ci, hi = c[:, i] * nd, h[:, i] * nd
            nb = self.nbr[i]
            if v in ('ia2c', 'ma2c_cu'):
                s = torch.relu(x[i] @ self._w(i, 'fc/w') + self._w(i, 'fc/b'))
                wx, wh, b = self._w(i, 'lstm/wx'), self._w(i, 'lstm/wh'), self._w(i, 'lstm/b')
            elif v == 'ia2c_fp':
                n_x = self.n_s_ls[i] - self.n_a * len(nb)
                # the environment attaches the fingerprints to the observation; tests that keep them in a
                # separate array pass observations of width n_x plus ps
                fp_in = x[i][:, n_x:] if x[i].shape[1] > n_x else cat([p[:, j] for j in nb])
                hx = torch.relu(x[i][:, :n_x] @ self._w(i, 'fcs/w') + self._w(i, 'fcs/b'))
                hp = torch.relu(fp_in @ self._w(i, 'fcp/w') + self._w(i, 'fcp/b'))
                s = torch.cat([hx, hp], dim=1)
                wx, wh, b = self._w(i, 'lstm/wx'), self._w(i, 'lstm/wh'), self._w(i, 'lstm/b')
            elif self.hetero and not nb:        # lstm_*_hetero, agent without neighbours: observation encoder only
                wx, wh, b = self._w(i, 'wx_hid'), self._w(i, 'wh_hid'), self._w(i, 'b_hid')
                act = torch.tanh if v == 'ma2c_ic3' else torch.relu
                s = act(x[i][:, :self.n_s_ls[i]] @ self._w(i, 'w_ob') + self._w(i, 'b_ob'))
            else:
                # hetero: every source contributes its own valid width (tf.slice(raw_xi, [j,0], [1, ns_dim]), :316-317)
                xi = torch.cat([x[i][:, :self.n_s_ls[i]]] + [x[j][:, :self.n_s_ls[j]] for j in nb], dim=1)
                wx, wh, b = self._w(i, 'wx_hid'), self._w(i, 'wh_hid'), self._w(i, 'b_hid')
                if v == 'ma2c_nc':
                    mi = cat([h[:, j] for j in nb])
                    pi_in = cat([p[:, j, :self.n_a_ls[j]] for j in nb])
                    hx = torch.relu(xi @ self._w(i, 'w_ob') + self._w(i, 'b_ob'))
                    hp = torch.relu(pi_in @ self._w(i, 'w_fp') + self._w(i, 'b_fp'))
                    hm = torch.relu(mi @ self._w(i, 'w_msg') + self._w(i, 'b_msg'))
                    s = torch.cat([hx, hp, hm], dim=1)
                elif v == 'ma2c_ic3':
                    mi = torch.stack([h[:, j] for j in nb], dim=0).mean(dim=0)
                    s = torch.tanh(xi @ self._w(i, 'w_ob') + self._w(i, 'b_ob')) + mi @ self._w(i, 'w_msg') + self._w(i, 'b_msg')
                else:  # dial
                    mi = cat([msg[j] for j in nb])
                    ai = torch.nn.functional.one_hot(torch.argmax(p[:, i], dim=1), self.n_h).to(self.dtype)
                    hx = torch.relu(xi @ self._w(i, 'w_ob') + self._w(i, 'b_ob'))
                    hm = torch.relu(mi @ self._w(i, 'w_msg') + self._w(i, 'b_msg'))
                    s = hx + hm + ai
            z = s @ wx + hi @ wh + b
            ig, fg, og, ug = torch.split(z, self.n_h, dim=1)
            ci = torch.sigmoid(fg) * ci + torch.sigmoid(ig) * torch.tanh(ug)
            hi = torch.sigmoid(og) * torch.tanh(ci)
            new_c.append(ci); new_h.append(hi)
        return torch.stack(new_c, dim=1), torch.stack(new_h, dim=1)

    def _pi(self, i, h):
        return torch.softmax(h @ self._head(i, 'pi/w') + self._head(i, 'pi/b'), dim=-1)

    def _pad_pi(self, pi):
        """hetero: zero-pad to the widest action space so policies stack; padded entries carry probability 0."""
        if pi.shape[-1] == self.n_a:
            return pi
        return torch.cat([pi, torch.zeros(*pi.shape[:-1], self.n_a - pi.shape[-1], dtype=pi.dtype)], dim=-1)

    def _v(self, i, h, actions):
        """actions [B,N] int64 (same-step actions); neighbours one-hot in ascending index."""
        parts = [h] + [torch.nn.functional.one_hot(actions[:, j], self.n_a_ls[j]).to(self.dtype) for j in self.nbr[i]]
        return (torch.cat(parts, dim=1) @ self._head(i, 'v/w') + self._head(i, 'v/b')).squeeze(-1)

    def _prep(self, obs, ps):
        x = [torch.as_tensor(np.asarray(o), dtype=self.dtype).reshape(self.B, -1) for o in obs]
        if ps is not None and self.hetero and not isinstance(ps, np.ndarray):      # list of per-agent [n_a_i] policies
            pad = np.zeros((self.B, self.N, self.n_a))
            for i, q in enumerate(ps):
                q = np.asarray(q, dtype=np.float64).reshape(self.B, -1)
                pad[:, i, :q.shape[1]] = q                                         # agents/models.py:229-235
            ps = pad
        p = None if ps is None else torch.as_tensor(np.asarray(ps), dtype=self.dtype).reshape(self.B, self.N, self.n_a)
        return x, p

    # ---- reference forward protocol (policies.py:119-134, 215-230) --------------------
    def forward(self, obs, done, ps=None, actions=None, out_type='p'):
        """obs: list of N arrays [B,n_s_i] (or [n_s_i] when B=1); done: scalar or [B];
        ps [B,N,n_a]; actions [B,N].  'p' stores the new state, 'v' does not (quirk Q1)."""
        with torch.no_grad():
            x, p = self._prep(obs, ps)
            d = torch.as_tensor(np.broadcast_to(np.asarray(done, dtype=np.float64), (self.B,)).copy(), dtype=self.dtype)
            c, h = self.states_fw[..., :self.n_h], self.states_fw[..., self.n_h:]
            c2, h2 = self._cell(x, p, d, c, h)
            if out_type.startswith('p'):
                self.states_fw = torch.cat([c2, h2], dim=-1)
                if self.hetero:                 # per-agent widths: a list like the reference's pi_ls (policies.py:296)
                    return [self._pi(i, h2[:, i]).numpy() for i in range(self.N)]
                return torch.stack([self._pi(i, h2[:, i]) for i in range(self.N)], dim=1).numpy()
            a = torch.as_tensor(np.asarray(actions), dtype=torch.int64).reshape(self.B, self.N)
            return torch.stack([self._v(i, h2[:, i], a) for i in range(self.N)], dim=1).numpy()

    # ---- training pass -----------------------------------------------------------------
    def unroll(self, obs, ps, acts, dones, state):
        """obs: list over t of (list of N [B,n_s_i]); ps [T,B,N,n_a]; acts [T,B,N]; dones [T,B] (pre-step).
        Returns pi [T,B,N,n_a], v [T,B,N]."""
        c, h = state[..., :self.n_h], state[..., self.n_h:]
        pis, vs = [], []
        T = len(obs)
        for t in range(T):
            x, p = self._prep(obs[t], None if ps is None else ps[t])
            d = torch.as_tensor(np.asarray(dones[t], dtype=np.float64).reshape(self.B), dtype=self.dtype)
            c, h = self._cell(x, p, d, c, h)
            a = torch.as_tensor(np.asarray(acts[t]), dtype=torch.int64).reshape(self.B, self.N)
            pis.append(torch.stack([self._pad_pi(self._pi(i, h[:, i])) for i in range(self.N)], dim=1))
            vs.append(torch.stack([self._v(i, h[:, i], a) for i in range(self.N)], dim=1))
        return torch.stack(pis), torch.stack(vs)

    def loss_terms(self, pi, v, acts, Rs, Advs, v_coef, e_coef):
        """policies.py:236-255; per-agent terms [N] (mean over (t,b))."""
        a = torch.as_tensor(np.asarray(acts), dtype=torch.int64)
        R = torch.as_tensor(np.asarray(Rs), dtype=self.dtype)
        A = torch.as_tensor(np.asarray(Advs), dtype=self.dtype)
        if self.hetero:
            # Reference quirk Q7 (agents/policies.py:241-251): in the non-identical branch prob_pi is built as
            # [N,1,T] and multiplied with ADV [N,T]; TF broadcasts that to [N,N,T], so after mean_t and the sum over
            # everything agent i's log-probability is weighted by the SUM over agents of the advantages.
            A = A.sum(dim=-1, keepdim=True).expand_as(A)
        log_pi = torch.log(torch.clamp(pi, 1e-10, 1.0))
        ent = -(pi * log_pi).sum(-1)                                  # [T,B,N]
        lp = torch.gather(log_pi, -1, a.unsqueeze(-1)).squeeze(-1)
        e_loss = -ent.mean(dim=(0, 1)) * e_coef
        p_loss = -(lp * A).mean(dim=(0, 1))
        v_loss = ((R - v) ** 2).mean(dim=(0, 1)) * 0.5 * v_coef
        return p_loss, v_loss, e_loss

    def consensus_update(self):
        """ConsensusPolicy._consensus_update (agents/policies.py:351-359, 401-426): every LSTM variable of
        agent i := mean over [i] + neighbours (ascending) of that variable.  The reference groups the assigns
        in one session.run without ordering them; the intended simultaneous update is restated here (all
        means are taken from the pre-update values)."""
        new = {}
        for i in range(self.N):
            agents = [i] + list(self.nbr[i])
            for key in ('wx', 'wh', 'b'):
                acc = self.p['cu/lstm_%da/%s' % (agents[0], key)].detach().clone()
                for j in agents[1:]:
                    acc = acc + self.p['cu/lstm_%da/%s' % (j, key)].detach()
                new['cu/lstm_%da/%s' % (i, key)] = acc / float(len(agents))
        for n, val in new.items():
            self.p[n].copy_(val)

    def _groups(self):
        if self.variant in ('ia2c', 'ia2c_fp'):      # one loss/clip/optimizer per agent (models.py:34-42)
            return [[n for n in self.names if n.startswith('lstm_%d/' % i)] for i in range(self.N)]
        return [self.names]

    def apply_grads(self, lr, max_grad_norm=40.0, alpha=0.99, epsilon=1e-5, apply=True):
        """clip_by_global_norm + TF RMSProp on ``self.grads`` (policies.py:34-39, 257-264); one group per agent for
        IA2C.  Returns the group norms.  Split out of ``backward`` so that tests can accumulate ``self.grads`` over
        env chunks of a large batch before the (single) optimizer step."""
        norms = []
        with torch.no_grad():
            for group in self._groups():
                gn = torch.sqrt(sum((self.grads[n] ** 2).sum() for n in group))
                norms.append(float(gn))
                scale = max_grad_norm / max(float(gn), max_grad_norm) if max_grad_norm > 0 else 1.0
                if apply:
                    for n in group:
                        g = self.grads[n] * scale
                        self.ms[n].mul_(alpha).add_((1 - alpha) * g * g)
                        self.p[n].sub_(lr * g / torch.sqrt(self.ms[n] + epsilon))
            if apply and self.variant == 'ma2c_cu':
                self.consensus_update()
        return norms

    def backward(self, obs, ps, acts, dones, Rs, Advs, lr, v_coef=0.5, e_coef=0.05,
                 max_grad_norm=40.0, alpha=0.99, epsilon=1e-5, apply=True):
        """Rs/Advs in [T,B,N] layout.  Returns dict of summaries; grads kept in self.grads."""
        for t in self.p.values():
            t.grad = None
        pi, v = self.unroll(obs, ps, acts, dones, self.states_bw)
        p_loss, v_loss, e_loss = self.loss_terms(pi, v, acts, Rs, Advs, v_coef, e_coef)
        loss = p_loss.sum() + v_loss.sum() + e_loss.sum()
        loss.backward()
        self.grads = {n: (self.p[n].grad.detach().clone() if self.p[n].grad is not None
                          else torch.zeros_like(self.p[n])) for n in self.names}
        norms = self.apply_grads(lr, max_grad_norm, alpha, epsilon, apply=apply)
        self.states_bw = self.states_fw.clone()
        self.last_pi, self.last_v = pi.detach(), v.detach()
        return dict(policy_loss=p_loss.detach().numpy(), value_loss=v_loss.detach().numpy(),
                    entropy_loss=e_loss.detach().numpy(), total_loss=float(loss.detach()), grad_norm=norms)
