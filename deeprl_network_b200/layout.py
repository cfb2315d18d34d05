"""Flat parameter layout + the `nmarl_model` descriptor handed to the kernels.

Variable names, shapes and creation order follow the reference graphs so checkpoints and the
parity tests can address weights by the reference's own names:
  NeurComm  nc/lstm_comm_i/{w_msg,b_msg,w_ob,b_ob,w_fp,b_fp,wx_hid,wh_hid,b_hid}  agents/utils.py:141-162
  CommNet   ic3/lstm_ic3_i/{w_msg,b_msg,w_ob,b_ob,wx_hid,wh_hid,b_hid}           agents/utils.py:361-377
  DIAL      dial/lstm_comm_i/{...}, dial/mfc_i/{w,b}                               agents/utils.py:535-566
  IA2C      lstm_i/fc/{w,b}, lstm_i/lstm/{wx,wh,b}                                 agents/policies.py:145-146
  IA2C_FP   lstm_i/fcs/{w,b}, lstm_i/fcp/{w,b}, lstm_i/lstm/{wx,wh,b}              agents/policies.py:157-185
  IA2C_CU   cu/fc_ia/{w,b}, cu/lstm_ia/{wx,wh,b}, cu/pi_i, cu/v_ia                 agents/policies.py:366-399
  heads     <scope>/pi_i/{w,b}, <scope>/v_i/{w,b}   (IA2C: lstm_i/pi, lstm_i/v)    agents/policies.py:50-77

Two agents reuse another agent's kernels (SURVEY 8 f2):
  ma2c_cu  runs the IA2C cell with the agent's OWN observation only (ob[i], n_s = 5) and one global clip.
  ia2c_fp  runs the NeurComm cell with a null message encoder: its [fcs | fcp] -> lstm network is the
           NeurComm cell whose w_msg / b_msg and wx_hid rows 128..191 are zero.  relu(0) = 0 feeds exact
           zeros into the gate GEMM and receives exact-zero gradients, so the padding never moves and
           the outputs equal FPPolicy's bit for bit.  The padding has no reference name and is not part
           of pack()/unpack()/checkpoints.

In the flat buffer every tensor starts on a 16-byte boundary, one agent's tensors are
contiguous (IA2C clips/optimises per agent) and wx_hid/wh_hid are adjacent so the LSTM gate
GEMM sees one [s_dim+n_h, 4*n_h] matrix.

Width: num_lstm = n_h in {16, 32, 64}.  The MA2C family and ma2c_cu size every encoder by n_h and ignore num_fc
(agents/policies.py:192, agents/models.py:103-104); ia2c / ia2c_fp need num_fc == num_lstm.
"""
import numpy as np

from . import _lib as L

VARIANT_ID = {'ia2c': L.IA2C, 'ma2c_nc': L.NC, 'ma2c_ic3': L.IC3, 'ma2c_dial': L.DIAL, 'ma2c_cu': L.IA2C, 'ia2c_fp': L.NC}
PER_AGENT_OPT = ('ia2c', 'ia2c_fp')        # one loss / clip / optimizer per agent (agents/models.py:34-42)
SCOPE = {'ma2c_nc': 'nc', 'ma2c_ic3': 'ic3', 'ma2c_dial': 'dial'}
CELL = {'ma2c_nc': 'lstm_comm', 'ma2c_ic3': 'lstm_ic3', 'ma2c_dial': 'lstm_comm'}
NH = L.NH             # default width; a layout's own width is ModelLayout.n_h


def _up4(x):
    return (int(x) + 3) // 4 * 4


SMEM_LIMIT = 227 * 1024    # dynamic shared memory one CTA can opt in to on sm_90 (bytes)


def ffma_fwd_smem_bytes(ld_in, s_dim, n_h):
    """Dynamic shared memory of the FP32-FFMA cell kernel (csrc/cell_fwd.cu: fwd_smem_floats with BM = 64, KC = 16):
    max(input tile, gate-weight ring, new-h tile) + [s | own h] tile + encoder-weight ring.  It is the only kernel
    whose shared memory grows with the observation width (DESIGN 4.8)."""
    bm, kc = 64, 16
    region0 = max(bm * ld_in, 2 * kc * 4 * n_h, bm * (n_h + 4))
    return 4 * (region0 + bm * (s_dim + n_h + 4) + 2 * kc * n_h)


def ortho_init(shape, scale=np.sqrt(2)):
    """Orthogonal init from the GLOBAL NumPy stream (agents/utils.py:10-23): tall matrices get
    orthonormal columns, wide ones orthonormal rows, times sqrt(2)."""
    a = np.random.standard_normal(shape)
    u, _, vt = np.linalg.svd(a, full_matrices=False)
    q = u if u.shape == tuple(shape) else vt
    return (scale * q.reshape(shape)).astype(np.float32)


class ModelLayout:
    def __init__(self, variant, n_s_ls, n_a, neighbor_mask, n_h=64, n_fc=64, obs_mode='gather', base_n_s=None):
        """obs_mode 'gather': the obs buffer holds each agent's OWN features (width base_n_s) and the
        kernel concatenates own + neighbours' rows (what the MA2C graphs do, and equal to the IA2C
        env observation).  'concat' (IA2C API mode): rows are the caller's pre-concatenated obs."""
        if variant not in VARIANT_ID:
            raise ValueError('unsupported agent %r (covered: ia2c, ia2c_fp, ma2c_cu, ma2c_nc, ma2c_ic3, ma2c_dial)' % variant)
        n_h, n_fc = int(n_h), int(n_fc)
        if n_h not in L.WIDTHS:
            raise ValueError('num_lstm = %d is not supported (kernels exist for %s)' % (n_h, ', '.join(map(str, L.WIDTHS))))
        if variant in ('ia2c', 'ia2c_fp') and n_fc != n_h:
            # the MA2C family and ma2c_cu size their encoders by num_lstm and ignore num_fc, as the reference does
            raise ValueError('%s needs num_fc == num_lstm (got num_fc = %d, num_lstm = %d)' % (variant, n_fc, n_h))
        self.n_h = n_h
        self.variant, self.vid = variant, VARIANT_ID[variant]
        mask = np.asarray(neighbor_mask).astype(int)
        N = len(mask)
        if N > L.MAX_AGENT:
            raise ValueError('n_agent %d > %d' % (N, L.MAX_AGENT))
        if not 0 < n_a < L.MAX_NA:
            raise ValueError('n_a %d out of range (1..%d actions)' % (n_a, L.MAX_NA - 1))
        self.N, self.n_a, self.mask = N, int(n_a), mask
        self.nbr = [list(map(int, np.where(mask[i] == 1)[0])) for i in range(N)]
        if max(len(x) for x in self.nbr) > L.MAX_NBR:
            raise ValueError('more than %d neighbours' % L.MAX_NBR)
        self.n_s_ls = [int(x) for x in n_s_ls]
        self.obs_mode = obs_mode
        self.concat = obs_mode == 'concat' and variant in ('ia2c', 'ia2c_fp')     # one source per agent, own width
        if variant == 'ia2c_fp' and obs_mode == 'concat':
            # heterogeneous agents (HeteroLayout): n_s_ls is the width of each agent's own pre-concatenated
            # observation, which feeds fcs; the fingerprints are still gathered per neighbour on the device
            assert getattr(self, 'hetero', False), 'ia2c_fp observations are gathered on the device'
            self.base_n_s = None
        elif variant == 'ia2c_fp':
            # n_s_ls counts own + neighbour observations + neighbour fingerprints (agents/models.py:175)
            assert obs_mode == 'gather', 'ia2c_fp observations are gathered on the device'
            self.base_n_s = int(base_n_s) if base_n_s else (self.n_s_ls[0] - n_a * len(self.nbr[0])) // (1 + len(self.nbr[0]))
            for i in range(N):
                assert self.n_s_ls[i] == (self.base_n_s + n_a) * len(self.nbr[i]) + self.base_n_s, 'ia2c_fp n_s_ls'
        elif variant == 'ia2c':
            if obs_mode == 'gather':
                self.base_n_s = int(base_n_s) if base_n_s else self.n_s_ls[0] // (1 + len(self.nbr[0]))
                for i in range(N):
                    assert self.n_s_ls[i] == self.base_n_s * (1 + len(self.nbr[i])), 'IA2C n_s_ls is not own+neighbours'
            else:
                self.base_n_s = None
        else:
            self.base_n_s = self.n_s_ls[0]
            assert all(x == self.base_n_s for x in self.n_s_ls), 'MA2C agents must share n_s'
        self.s_dim = 3 * n_h if variant in ('ma2c_nc', 'ia2c_fp') else n_h
        self._build()

    # ------------------------------------------------------------------------------------------
    def _kx(self, i):
        if self.concat:
            return self.n_s_ls[i]
        if self.variant == 'ma2c_cu':
            return self.base_n_s
        return self.base_n_s * (1 + len(self.nbr[i]))

    def _build(self):
        N, n_a, v, NH = self.N, self.n_a, self.variant, self.n_h
        self.entries = []          # (reference name, offset, shape)
        self.agents_off = []
        off = 0
        toff = 0
        poff = 0

        def put(name, shape):
            nonlocal off
            o = off
            self.entries.append((name, o, tuple(shape)))
            off = _up4(off + int(np.prod(shape)))
            return o

        def skip(n):                # unnamed zero padding (see the module docstring)
            nonlocal off
            o = off
            off = _up4(off + int(n))
            return o

        for i in range(N):
            nm = len(self.nbr[i])
            a = dict(p_begin=off)
            for k in ('o_w_ob', 'o_b_ob', 'o_w_fp', 'o_b_fp', 'o_w_msg', 'o_b_msg', 'o_wxh', 'o_b',
                      'o_mfc_w', 'o_mfc_b', 'o_pi_w', 'o_pi_b', 'o_v_w', 'o_v_b', 't_wxh', 't_w_msg', 't_mfc',
                      'tp_x', 'tp_p', 'tp_m', 'tp_g', 'tp_mfc', 'tp_gT', 'tp_mT', 'tp_mfcT'):
                a[k] = -1
            kx = self._kx(i)
            if v == 'ia2c':
                s = 'lstm_%d' % i
                a['o_w_ob'] = put(s + '/fc/w', (kx, NH)); a['o_b_ob'] = put(s + '/fc/b', (NH,))
                a['o_wxh'] = put(s + '/lstm/wx', (NH, 4 * NH))
                o2 = put(s + '/lstm/wh', (NH, 4 * NH)); assert o2 == a['o_wxh'] + NH * 4 * NH
                a['o_b'] = put(s + '/lstm/b', (4 * NH,))
                hp, hv = s + '/pi', s + '/v'
            elif v == 'ma2c_cu':
                a['o_w_ob'] = put('cu/fc_%da/w' % i, (kx, NH)); a['o_b_ob'] = put('cu/fc_%da/b' % i, (NH,))
                a['o_wxh'] = put('cu/lstm_%da/wx' % i, (NH, 4 * NH))
                o2 = put('cu/lstm_%da/wh' % i, (NH, 4 * NH)); assert o2 == a['o_wxh'] + NH * 4 * NH
                a['o_b'] = put('cu/lstm_%da/b' % i, (4 * NH,)); assert a['o_b'] == o2 + NH * 4 * NH
                hp, hv = 'cu/pi_%d' % i, 'cu/v_%da' % i
            elif v == 'ia2c_fp':
                s = 'lstm_%d' % i
                a['o_w_msg'] = skip(NH * nm * NH); a['o_b_msg'] = skip(NH)
                a['o_w_ob'] = put(s + '/fcs/w', (kx, NH)); a['o_b_ob'] = put(s + '/fcs/b', (NH,))
                a['o_w_fp'] = put(s + '/fcp/w', (n_a * nm, NH)); a['o_b_fp'] = put(s + '/fcp/b', (NH,))
                a['o_wxh'] = put(s + '/lstm/wx', (2 * NH, 4 * NH))
                o1 = skip(NH * 4 * NH); assert o1 == a['o_wxh'] + 2 * NH * 4 * NH
                o2 = put(s + '/lstm/wh', (NH, 4 * NH)); assert o2 == a['o_wxh'] + self.s_dim * 4 * NH
                a['o_b'] = put(s + '/lstm/b', (4 * NH,))
                hp, hv = s + '/pi', s + '/v'
                a['t_w_msg'] = toff; toff += _up4(NH * NH * nm)
            else:
                s = '%s/%s_%d' % (SCOPE[v], CELL[v], i)
                km = NH if v == 'ma2c_ic3' else NH * nm
                a['o_w_msg'] = put(s + '/w_msg', (km, NH)); a['o_b_msg'] = put(s + '/b_msg', (NH,))
                a['o_w_ob'] = put(s + '/w_ob', (kx, NH)); a['o_b_ob'] = put(s + '/b_ob', (NH,))
                if v == 'ma2c_nc':
                    a['o_w_fp'] = put(s + '/w_fp', (n_a * nm, NH)); a['o_b_fp'] = put(s + '/b_fp', (NH,))
                a['o_wxh'] = put(s + '/wx_hid', (self.s_dim, 4 * NH))
                o2 = put(s + '/wh_hid', (NH, 4 * NH)); assert o2 == a['o_wxh'] + self.s_dim * 4 * NH
                a['o_b'] = put(s + '/b_hid', (4 * NH,))
                if v == 'ma2c_dial':
                    a['o_mfc_w'] = put('dial/mfc_%d/w' % i, (NH, NH)); a['o_mfc_b'] = put('dial/mfc_%d/b' % i, (NH,))
                hp, hv = '%s/pi_%d' % (SCOPE[v], i), '%s/v_%d' % (SCOPE[v], i)
                a['t_w_msg'] = toff; toff += _up4(NH * km)
                if v == 'ma2c_dial':
                    a['t_mfc'] = toff; toff += NH * NH
            a['o_pi_w'] = put(hp + '/w', (NH, n_a)); a['o_pi_b'] = put(hp + '/b', (n_a,))
            a['o_v_w'] = put(hv + '/w', (NH + n_a * nm, 1)); a['o_v_b'] = put(hv + '/b', (1,))
            a['t_wxh'] = toff; toff += 4 * NH * (self.s_dim + NH)
            a['p_end'] = off
            # packed tensor-core operands: ceil(K/32) k-blocks x [hi|lo] x (N rows x 32 floats)
            def tp(K, N):
                nonlocal poff
                o = poff
                poff += ((K + 31) // 32) * 2 * N * 32
                return o
            a['tp_x'] = tp(kx, NH)
            if self.vid == L.NC:
                a['tp_p'] = tp(n_a * nm, NH)
            if self.vid != L.IA2C:
                km2 = NH if v == 'ma2c_ic3' else NH * nm
                a['tp_m'] = tp(km2, NH)
                a['tp_mT'] = tp(NH, km2)
            a['tp_g'] = tp(self.s_dim + NH, 4 * NH)
            a['tp_gT'] = tp(4 * NH, self.s_dim + NH)
            if v == 'ma2c_dial':
                a['tp_mfc'] = tp(NH, NH)
                a['tp_mfcT'] = tp(NH, NH)
            self.agents_off.append(a)
        self.n_param, self.n_wt, self.n_wp = off, max(toff, 4), max(poff, 4)
        self.kx_pad = _up4(max(self._kx(i) for i in range(N)))
        max_nbr = max(len(x) for x in self.nbr)
        self.kp_pad = _up4(n_a * max_nbr) if self.vid == L.NC else 0
        self.km_pad = {'ia2c': 0, 'ma2c_cu': 0, 'ma2c_ic3': NH}.get(v, NH * max_nbr)
        self.ld_in = self.kx_pad + self.kp_pad + self.km_pad
        smem = ffma_fwd_smem_bytes(self.ld_in, self.s_dim, NH)
        if smem > SMEM_LIMIT:
            # every model can meet the FFMA kernel (B not a multiple of 128, greedy evaluation); nmarl_policy_step_*
            # would refuse the launch with the same numbers
            raise ValueError('observation encoder too wide: %d gathered inputs per agent (x %d + fingerprints %d + '
                             'messages %d) need %d B of shared memory in the cell kernel, the limit is %d B'
                             % (self.ld_in, self.kx_pad, self.kp_pad, self.km_pad, smem, SMEM_LIMIT))
        if self.concat:
            self.obs_stride = _up4(max(self.n_s_ls))
        else:
            self.obs_stride = _up4(self.base_n_s)
        self.by_name = {n: (o, s) for n, o, s in self.entries}

    def c_model(self):
        m = L.Model()
        m.variant, m.n_agent, m.n_a, m.s_dim = self.vid, self.N, self.n_a, self.s_dim       # s_dim carries n_h
        m.obs_stride, m.kx_pad, m.kp_pad, m.km_pad = self.obs_stride, self.kx_pad, self.kp_pad, self.km_pad
        m.n_param, m.n_wt, m.n_wp = self.n_param, self.n_wt, self.n_wp
        m.per_agent_norm = 1 if self.variant in PER_AGENT_OPT else 0
        recv = [[] for _ in range(self.N)]
        for k in range(self.N):
            for slot, j in enumerate(self.nbr[k]):
                recv[j].append((k, slot))
        for i in range(self.N):
            ag = m.agent[i]
            ag.n_nbr = len(self.nbr[i])
            for s, j in enumerate(self.nbr[i]):
                ag.nbr[s] = j
            if len(recv[i]) > L.MAX_NBR:
                raise ValueError('agent %d is a neighbour of more than %d agents' % (i, L.MAX_NBR))
            ag.n_recv = len(recv[i])
            for s, (k, slot) in enumerate(recv[i]):
                ag.recv_agent[s], ag.recv_slot[s] = k, slot
            if self.concat:
                ag.x_nsrc, ag.x_w = 1, self.n_s_ls[i]
                ag.x_src[0] = i
            else:
                srcs = [i] if self.variant == 'ma2c_cu' else [i] + self.nbr[i]
                ag.x_nsrc, ag.x_w = len(srcs), self.base_n_s
                for s, j in enumerate(srcs):
                    ag.x_src[s] = j
            for k, val in self.agents_off[i].items():
                setattr(ag, k, val)
        return m

    # ---- host-side packing -----------------------------------------------------------------------
    def init_flat(self):
        """Reference initialisation order (SURVEY A.5): consumes np.random like graph construction."""
        params = {}
        for name, shape in self.creation_order():
            params[name] = ortho_init(shape) if len(shape) == 2 else np.zeros(shape, dtype=np.float32)
        return self.pack(params)

    def creation_order(self):
        """(name, shape) in tf.get_variable order: cells for all agents, (DIAL: mfc), then heads;
        IA2C agent by agent."""
        v, N = self.variant, self.N
        shapes = {n: s for n, _, s in self.entries}
        order = []
        if v == 'ia2c':
            for i in range(N):
                s = 'lstm_%d' % i
                order += [s + '/fc/w', s + '/fc/b', s + '/lstm/wx', s + '/lstm/wh', s + '/lstm/b',
                          s + '/pi/w', s + '/pi/b', s + '/v/w', s + '/v/b']
        elif v == 'ia2c_fp':            # fcs, fcp, lstm, heads per policy (agents/policies.py:173-185)
            for i in range(N):
                s = 'lstm_%d' % i
                order += [s + '/fcs/w', s + '/fcs/b', s + '/fcp/w', s + '/fcp/b', s + '/lstm/wx', s + '/lstm/wh',
                          s + '/lstm/b', s + '/pi/w', s + '/pi/b', s + '/v/w', s + '/v/b']
        elif v == 'ma2c_cu':            # agent by agent inside one graph (agents/policies.py:378-396)
            for i in range(N):
                order += ['cu/fc_%da/w' % i, 'cu/fc_%da/b' % i, 'cu/lstm_%da/wx' % i, 'cu/lstm_%da/wh' % i,
                          'cu/lstm_%da/b' % i, 'cu/pi_%d/w' % i, 'cu/pi_%d/b' % i, 'cu/v_%da/w' % i, 'cu/v_%da/b' % i]
        else:
            for i in range(N):
                s = '%s/%s_%d' % (SCOPE[v], CELL[v], i)
                order += [s + '/w_msg', s + '/b_msg', s + '/w_ob', s + '/b_ob']
                if v == 'ma2c_nc':
                    order += [s + '/w_fp', s + '/b_fp']
                order += [s + '/wx_hid', s + '/wh_hid', s + '/b_hid']
            if v == 'ma2c_dial':
                for i in range(N):
                    order += ['dial/mfc_%d/w' % i, 'dial/mfc_%d/b' % i]
            for i in range(N):
                sc = SCOPE[v]
                order += ['%s/pi_%d/w' % (sc, i), '%s/pi_%d/b' % (sc, i), '%s/v_%d/w' % (sc, i), '%s/v_%d/b' % (sc, i)]
        return [(n, shapes[n]) for n in order]

    def pack(self, params):
        flat = np.zeros(self.n_param, dtype=np.float32)
        for name, o, shape in self.entries:
            a = np.asarray(params[name], dtype=np.float32)
            assert a.shape == shape, (name, a.shape, shape)
            flat[o:o + a.size] = a.ravel()
        return flat

    def unpack(self, flat):
        flat = np.asarray(flat)
        return {name: flat[o:o + int(np.prod(shape))].reshape(shape).copy() for name, o, shape in self.entries}

    def n_real_param(self):
        return int(sum(np.prod(s) for _, _, s in self.entries))


PI_PAD_BIAS = -1.0e30      # bias of a padded (non-existent) action: softmax gives it probability exactly 0


class HeteroLayout(ModelLayout):
    """Agents with UNEQUAL observation / action widths (the reference's ``identical_agent == False`` path:
    lstm_comm_hetero / lstm_ic3_hetero / lstm_dial_hetero, agents/utils.py:220-341, 420-512, 602-702; per-agent
    heads, agents/policies.py:59-77, 289-312, 386; zero-padded inputs, agents/models.py:229-235; per-agent
    LstmPolicy / FPPolicy with per-neighbour action widths, agents/models.py:118-132, 171-188).

    The kernels stay homogeneous: the model is EMBEDDED in a padded one with ``n_s = max(n_s_ls)`` and
    ``n_a = max(n_a_ls)`` for everybody.  Every reference tensor (tight shape, reference name, reference creation
    order) maps onto a sub-block of the padded tensor; the rest of the padded tensor is zero and provably stays zero:
      * padded observation / fingerprint inputs are 0, so the weight rows they meet get gradient x^T d = 0;
      * a padded action has policy-head bias PI_PAD_BIAS and zero weights -> pi = exp(-1e30 - max) = 0 exactly,
        d(logit) = pi * (g - <pi, g>) = 0, it is never sampled (its cdf step has zero width) and never the arg-max;
      * value-head rows of padded actions are never selected by a one-hot;
      * an agent without neighbours keeps zero message / fingerprint encoders (relu(0) = 0 feeds the gate GEMM
        zeros and receives zero gradients -- the same argument as for ia2c_fp, see the module docstring); a DIAL
        one also drops the one-hot of its own last action (o_b_msg = -1), as lstm_dial_hetero does.
    Zero gradients leave clip-by-global-norm and RMSProp untouched, so pi, v, gradients and trained weights equal
    the reference's tight model.  pack / unpack / creation_order / checkpoints speak the reference's tight tensors.

    Per variant:
      * ma2c_nc / ma2c_ic3 / ma2c_dial: observations padded to n_s_max, gathered from the agent and its neighbours.
      * ia2c / ia2c_fp: every agent reads the caller's own pre-concatenated observation of width n_s_ls[i]
        (x_nsrc = 1, x_w = n_s_ls[i]; for ia2c_fp that is the part in front of the fingerprints, which feeds fcs), so
        fc / fcs need no padding.  ia2c_fp gathers the neighbours' fingerprints, each n_a_max wide: fcp row
        k * n_a_max + a is action a of the k-th neighbour.  An ia2c_fp agent without neighbours has no fcp and a
        [64, 256] lstm/wx (rows 64..127 of the padded one, and b_fp, are padding).
      * ma2c_cu: ConsensusPolicy pads every observation to n_s_max and fc_%da acts on the padded width, so its
        tight fc_%da/w is the whole [n_s_max, 64] tensor.  Its policy head is named cu/pi_%da (agents/policies.py:386).
    """

    def __init__(self, variant, n_s_ls, n_a_ls, neighbor_mask, n_h=64, n_fc=64):
        if variant not in VARIANT_ID:
            raise ValueError('unsupported agent %r' % variant)
        self.tight_n_s, self.tight_n_a = [int(x) for x in n_s_ls], [int(x) for x in n_a_ls]
        ns_max, na_max = max(self.tight_n_s), max(self.tight_n_a)
        self.hetero = True
        if variant in PER_AGENT_OPT:
            super().__init__(variant, self.tight_n_s, na_max, neighbor_mask, n_h=n_h, n_fc=n_fc, obs_mode='concat')
        else:
            super().__init__(variant, [ns_max] * len(self.tight_n_s), na_max, neighbor_mask, n_h=n_h, n_fc=n_fc,
                             obs_mode='gather')
        if variant == 'ma2c_ic3' and min(len(x) for x in self.nbr) == 0:
            raise NotImplementedError('CommNet agent without neighbours (mean over an empty set) is not supported')
        if variant == 'ma2c_dial':
            # lstm_dial_hetero gives an agent without neighbours s = relu(x w_ob + b_ob) alone: no message term and no
            # one-hot of its own last action (agents/utils.py:683-685).  The kernels drop both when o_b_msg = -1.
            for i in range(self.N):
                if not self.nbr[i]:
                    self.agents_off[i]['o_b_msg'] = -1
        self._embed()

    def _embed(self):
        v, N, ns_max, na_max, NH = self.variant, self.N, self.base_n_s, self.n_a, self.n_h
        pad = {n: (o, s) for n, o, s in self.entries}           # padded tensors of the inner homogeneous layout
        tight, idx = [], {}

        def rows(name, new_name, row_ids, ncol):
            """tight tensor = the listed rows of padded tensor `name` (all `ncol` columns)."""
            o, shp = pad[name]
            pc = shp[1] if len(shp) == 2 else 1
            r = np.asarray(row_ids, dtype=np.int64)
            idx[new_name] = (o + r[:, None] * pc + np.arange(ncol)[None, :]).ravel()
            tight.append((new_name, (len(r), ncol)))

        def vec(name, n=None, new_name=None):
            o, shp = pad[name]
            n = shp[0] if n is None else n
            new_name = new_name or name
            idx[new_name] = o + np.arange(n, dtype=np.int64)
            tight.append((new_name, (n,)))

        self.pi_pad = []

        def heads(i, hp, hv, tight_hp=None):
            """the agent's n_a_i policy columns (padded actions get PI_PAD_BIAS); value head: h, then one one-hot
            block per neighbour j with its n_a_j real rows at stride n_a_max"""
            tight_hp = tight_hp or hp
            na = self.tight_n_a[i]
            o, _ = pad[hp + '/w']
            idx[tight_hp + '/w'] = (o + np.arange(NH)[:, None] * na_max + np.arange(na)[None, :]).ravel()
            tight.append((tight_hp + '/w', (NH, na)))
            vec(hp + '/b', na, tight_hp + '/b')
            ob, _ = pad[hp + '/b']
            self.pi_pad += [ob + a for a in range(na, na_max)]
            v_rows = list(range(NH)) + [NH + k * na_max + a for k, j in enumerate(self.nbr[i]) for a in range(self.tight_n_a[j])]
            rows(hv + '/w', hv + '/w', v_rows, 1); vec(hv + '/b')

        if v in PER_AGENT_OPT or v == 'ma2c_cu':
            # one policy after the other, each with its own heads (agents/policies.py:136-185, 378-396)
            for i in range(N):
                nb = self.nbr[i]
                if v == 'ma2c_cu':
                    s = 'cu/'
                    rows(s + 'fc_%da/w' % i, s + 'fc_%da/w' % i, range(ns_max), NH); vec(s + 'fc_%da/b' % i)
                    lstm = s + 'lstm_%da' % i
                else:
                    s = 'lstm_%d/' % i
                    enc = 'fc' if v == 'ia2c' else 'fcs'
                    rows(s + enc + '/w', s + enc + '/w', range(self.tight_n_s[i]), NH); vec(s + enc + '/b')
                    if v == 'ia2c_fp' and nb:
                        p_rows = [k * na_max + a for k, j in enumerate(nb) for a in range(self.tight_n_a[j])]
                        rows(s + 'fcp/w', s + 'fcp/w', p_rows, NH); vec(s + 'fcp/b')
                    lstm = s + 'lstm'
                n_in = 2 * NH if (v == 'ia2c_fp' and nb) else NH
                rows(lstm + '/wx', lstm + '/wx', range(n_in), 4 * NH)
                rows(lstm + '/wh', lstm + '/wh', range(NH), 4 * NH); vec(lstm + '/b')
                if v == 'ma2c_cu':
                    heads(i, 'cu/pi_%d' % i, 'cu/v_%da' % i, tight_hp='cu/pi_%da' % i)
                else:
                    heads(i, s + 'pi', s + 'v')
        else:
            sc, cell = SCOPE[v], CELL[v]
            for i in range(N):
                s = '%s/%s_%d' % (sc, cell, i)
                nb = self.nbr[i]
                x_rows = [f for f in range(self.tight_n_s[i])] + [(k + 1) * ns_max + f for k, j in enumerate(nb) for f in range(self.tight_n_s[j])]
                p_rows = [k * na_max + a for k, j in enumerate(nb) for a in range(self.tight_n_a[j])]
                km = NH if v == 'ma2c_ic3' else NH * len(nb)
                if v == 'ma2c_nc':           # creation order of lstm_comm_hetero: w_ob first (agents/utils.py:260-283)
                    rows(s + '/w_ob', s + '/w_ob', x_rows, NH); vec(s + '/b_ob')
                    if nb:
                        rows(s + '/w_fp', s + '/w_fp', p_rows, NH); vec(s + '/b_fp')
                        rows(s + '/w_msg', s + '/w_msg', range(km), NH); vec(s + '/b_msg')
                    rows(s + '/wx_hid', s + '/wx_hid', range(3 * NH if nb else NH), 4 * NH)
                else:
                    if nb:
                        rows(s + '/w_msg', s + '/w_msg', range(km), NH); vec(s + '/b_msg')
                    rows(s + '/w_ob', s + '/w_ob', x_rows, NH); vec(s + '/b_ob')
                    rows(s + '/wx_hid', s + '/wx_hid', range(NH), 4 * NH)
                rows(s + '/wh_hid', s + '/wh_hid', range(NH), 4 * NH); vec(s + '/b_hid')
            if v == 'ma2c_dial':
                for i in range(N):
                    rows('dial/mfc_%d/w' % i, 'dial/mfc_%d/w' % i, range(NH), NH); vec('dial/mfc_%d/b' % i)
            for i in range(N):
                heads(i, '%s/pi_%d' % (sc, i), '%s/v_%d' % (sc, i))
        self._idx, self._tight = idx, tight
        self._tight_shapes = dict(tight)
        # `entries` is what callers enumerate (names, shapes, checkpoints): reference tensors; offset = first element
        self.entries = [(n, int(idx[n][0]) if len(idx[n]) else 0, s) for n, s in tight]
        self.by_name = {n: (o, s) for n, o, s in self.entries}

    def creation_order(self):
        return list(self._tight)          # built in tf.get_variable order

    def pack(self, params):
        flat = np.zeros(self.n_param, dtype=np.float32)
        flat[self.pi_pad] = PI_PAD_BIAS
        for name, shape in self._tight:
            a = np.asarray(params[name], dtype=np.float32)
            assert a.shape == shape, (name, a.shape, shape)
            flat[self._idx[name]] = a.ravel()
        return flat

    def unpack(self, flat):
        flat = np.asarray(flat)
        return {name: flat[self._idx[name]].reshape(shape).copy() for name, shape in self._tight}

    def n_real_param(self):
        return int(sum(np.prod(s) for _, s in self._tight))
