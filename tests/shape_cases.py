"""The shape envelope both tests/test_shape_envelope.py (host) and tests/test_gpu_shapes.py (device) walk: observation
widths, action counts and neighbour counts around every edge of the cell kernels, far outside the CACC shapes
(n_s = 5, n_a = 4) the other parity tests use.  The observation encoder contracts over K = n_s * (1 + neighbours)
inputs (n_s alone for ma2c_cu, the agent's own width for pre-concatenated IA2C observations); the tensor-core kernels
take K <= 32 (one 32-deep k-block), the FP32-FFMA kernels walk any K in 16-deep chunks.

Each case: variant, topology, own-observation width n_s (a list: pre-concatenated IA2C observations of unequal width),
n_a, and `tc`, the kernel family that must run it when the env count is a multiple of 128."""
import collections

import numpy as np

from oracle.cacc import chain_masks

Case = collections.namedtuple('Case', 'variant topo n_s n_a tc why')
VARIANTS = ['ma2c_nc', 'ma2c_ic3', 'ma2c_dial', 'ia2c', 'ia2c_fp', 'ma2c_cu']
CUT = 3                                   # topo 'cut8': the agent without neighbours
CASES = collections.OrderedDict()


def _add(variant, topo, n_s, n_a, tc, why):
    tag = 'concat%d' % max(n_s) if isinstance(n_s, list) else 's%d' % n_s
    CASES['%s-%s-%s-a%d' % (variant, topo, tag, n_a)] = Case(variant, topo, n_s, n_a, tc, why)


for _na in (1, 2, 3, 5, 6, 7):
    for _v in VARIANTS:
        _add(_v, 'chain8', 5, _na, True, 'generic-n_a heads; alignment padding behind pi/w, pi/b, v/w; n_a = 1: pi == 1')
for _v in ('ma2c_nc', 'ia2c_fp'):
    _add(_v, 'grid5', 5, 7, True, 'widest fingerprint encoder (K_fp = 28) and value-head one-hot block (64 + 28 rows)')
for _v in ('ma2c_nc', 'ma2c_ic3', 'ma2c_dial', 'ia2c'):
    _add(_v, 'chain8', 1, 4, True, 'K = 2..3: a single partly filled wgmma k-step')
    _add(_v, 'chain8', 8, 4, True, 'K = 16 / 24: whole k-steps')
    _add(_v, 'chain8', 10, 4, True, 'K = 30: the last k-step of the k-block is partly padding')
    _add(_v, 'chain8', 11, 4, False, 'K = 33: first width past the tensor-core kernels; 3 FFMA chunks, ragged last one')
    _add(_v, 'chain8', 20, 4, False, 'K = 60: 4 FFMA chunks')
for _v in ('ma2c_nc', 'ia2c'):
    _add(_v, 'ladder8', 8, 4, True, 'K = 32 exactly for the inner agents, 24 for the corners')
for _v in ('ma2c_nc', 'ia2c_fp'):
    _add(_v, 'grid5', 12, 5, False, 'a traffic-signal-like shape: 25 agents, K = 36..60, n_a = 5')
for _ns, _tc in ((31, True), (32, True), (33, False)):
    _add('ma2c_cu', 'chain8', _ns, 4, _tc, 'single-source encoder across the K = 32 boundary')
_add('ia2c', 'chain8', [32, 7, 12, 29, 30, 31, 5, 1], 4, True, 'pre-concatenated observations, widest exactly 32')
_add('ia2c', 'chain8', [33, 7, 12, 29, 30, 31, 5, 1], 4, False, 'pre-concatenated observations, widest 33')
for _v in ('ma2c_nc', 'ma2c_dial'):
    _add(_v, 'cut8', 11, 3, False, 'agent without neighbours (zero-width fingerprint / message operands) on the wide FFMA path')


def mask_of(topo):
    from gpu_common import cut_chain_mask, ladder_masks
    if topo == 'grid5':
        r, c = np.divmod(np.arange(25), 5)
        return ((np.abs(r[:, None] - r[None, :]) + np.abs(c[:, None] - c[None, :])) == 1).astype(int)
    return {'chain8': lambda: chain_masks(8)[0], 'ladder8': lambda: ladder_masks(4), 'cut8': lambda: cut_chain_mask(8, CUT)}[topo]()


def n_s_ls_of(case, mask):
    from gpu_common import widths
    return list(case.n_s) if isinstance(case.n_s, list) else widths(case.variant, mask, case.n_s, case.n_a)


def layout_of(case):
    from deeprl_network_b200.layout import ModelLayout
    mask = mask_of(case.topo)
    return ModelLayout(case.variant, n_s_ls_of(case, mask), case.n_a, mask,
                       obs_mode='concat' if isinstance(case.n_s, list) else 'gather')
