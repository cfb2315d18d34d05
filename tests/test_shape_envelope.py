"""Host side of the shape envelope (tests/shape_cases.py): the layout of every case is what the formulas say, packing
round-trips with zero padding, each case selects the kernel family the table states, and the widest observation the
cell kernels have shared memory for is known, enforced by ModelLayout, and equal to what the CUDA source computes."""
import numpy as np
import pytest

from helpers import random_params
from shape_cases import CASES, layout_of, mask_of, n_s_ls_of

NH = 64


def up4(x):
    return (x + 3) // 4 * 4


@pytest.mark.parametrize('cid', list(CASES))
def test_layout_of_case(cid):
    from deeprl_network_b200.agents.engine import tc_eligible
    c = CASES[cid]
    lay = layout_of(c)
    mask = mask_of(c.topo)
    nbr = [int(k) for k in mask.sum(1)]
    concat = isinstance(c.n_s, list)
    fam_nc = c.variant in ('ma2c_nc', 'ia2c_fp')
    if concat:
        kx = list(c.n_s)
    elif c.variant == 'ma2c_cu':
        kx = [c.n_s] * len(mask)
    else:
        kx = [c.n_s * (1 + k) for k in nbr]
    km = {'ia2c': [0] * len(mask), 'ma2c_cu': [0] * len(mask), 'ma2c_ic3': [NH] * len(mask)}.get(c.variant, [NH * k for k in nbr])
    assert lay.kx_pad == up4(max(kx))
    assert lay.kp_pad == (up4(c.n_a * max(nbr)) if fam_nc else 0)
    assert lay.km_pad == max(km)
    assert lay.obs_stride == up4(max(c.n_s) if concat else c.n_s)
    assert lay.ld_in == lay.kx_pad + lay.kp_pad + lay.km_pad
    # packed tensor-core operands: ceil(K / 32) k-blocks x [hi | lo] x (columns x 32 floats) per GEMM operand
    blk = lambda K, cols: -(-K // 32) * 2 * cols * 32
    s_dim = 3 * NH if fam_nc else NH
    n_wp = 0
    for i in range(len(mask)):
        n_wp += blk(kx[i], NH) + blk(s_dim + NH, 4 * NH) + blk(4 * NH, s_dim + NH)
        if fam_nc:
            n_wp += blk(c.n_a * nbr[i], NH)
        if c.variant not in ('ia2c', 'ma2c_cu'):
            n_wp += blk(km[i], NH) + blk(NH, km[i])
        if c.variant == 'ma2c_dial':
            n_wp += 2 * blk(NH, NH)
    assert lay.n_wp == n_wp
    # the model descriptor carries the same gather: x_nsrc sources of x_w columns each
    m = lay.c_model()
    for i in range(len(mask)):
        assert m.agent[i].x_nsrc * m.agent[i].x_w == kx[i] <= m.kx_pad
    # every tensor starts on a 16-byte boundary; pack / unpack round-trip; the floats between tensors are zero
    params = random_params(lay.creation_order(), seed=1)
    flat = lay.pack(params)
    back = lay.unpack(flat)
    used = np.zeros(lay.n_param, bool)
    for n, o, s in lay.entries:
        assert o % 4 == 0, n
        assert not used[o:o + int(np.prod(s))].any(), (n, 'overlaps another tensor')
        used[o:o + int(np.prod(s))] = True
        np.testing.assert_array_equal(back[n], params[n])
    assert n_s_ls_of(c, mask) == lay.n_s_ls
    assert used.sum() == lay.n_real_param() and np.all(flat[~used] == 0)
    if c.n_a % 4 and c.variant != 'ia2c_fp':
        assert (~used).any(), 'n_a % 4 != 0 leaves alignment padding behind pi/w, pi/b and v/w'
    # kernel family at B = 128, and never the tensor-core one on ragged env counts
    assert tc_eligible(lay, 128) == c.tc, (lay.kx_pad, lay.kp_pad)
    assert tc_eligible(lay, 256) == c.tc
    assert not tc_eligible(lay, 7) and not tc_eligible(lay, 130)


def test_table_reaches_every_edge():
    """The edges the table is there for, stated on the layouts themselves."""
    lays = {cid: layout_of(c) for cid, c in CASES.items()}
    kx_tc = {l.kx_pad for cid, l in lays.items() if CASES[cid].tc}
    kx_ffma = {l.kx_pad for cid, l in lays.items() if not CASES[cid].tc}
    assert max(kx_tc) == 32 and min(kx_ffma) == 36 and 4 in kx_tc
    assert {CASES[cid].n_a for cid in lays} == {1, 2, 3, 4, 5, 6, 7}
    raw_k = {c.n_s * 3 for c in CASES.values() if not isinstance(c.n_s, list) and c.topo == 'chain8' and c.variant == 'ma2c_nc'}
    assert {30, 33, 60} <= raw_k                       # partly padded last k-step; first FFMA fallback; 4 FFMA chunks
    assert any(l.kp_pad == 28 and l.N == 25 for l in lays.values())
    lad = lays['ma2c_nc-ladder8-s8-a4']
    assert sorted({len(x) for x in lad.nbr}) == [2, 3] and lad.kx_pad == 32
    assert any(l.kx_pad > 32 and min(len(x) for x in l.nbr) == 0 for l in lays.values())


def test_path_needs_the_tensor_core_width():
    from deeprl_network_b200.agents.engine import tc_eligible
    from deeprl_network_b200.layout import ModelLayout
    mask = mask_of('chain8')
    assert tc_eligible(ModelLayout('ma2c_nc', [5] * 8, 4, mask), 128)
    assert not tc_eligible(ModelLayout('ma2c_nc', [5] * 8, 4, mask, n_h=32, n_fc=32), 128)


# ---- shared-memory ceiling ---------------------------------------------------------------------------------------
SMEM_LIMIT = 227 * 1024


def fwd_smem_bytes(ld_in, s_dim, H=NH, BM=64, KC=16):
    """csrc/cell_fwd.cu: fwd_region0_floats + fwd_smem_floats (FWD_BM = 64, KC = 16)"""
    region0 = max(BM * ld_in, 2 * KC * 4 * H, BM * (H + 4))
    return 4 * (region0 + BM * (s_dim + H + 4) + 2 * KC * H)


def bwd_smem_bytes(ngrp, H=NH, BM=64):
    """csrc/train.cu: launch_bwd (BWD_BM = 64); NGRP = 4 for NeurComm, 2 otherwise"""
    return 4 * (BM * (4 * H + 4) + 2 * 16 * H * ngrp)


def wgrad_smem_bytes(nd):
    """csrc/train.cu: launch_wgrad, nd output columns"""
    return 4 * (2 * 32 * 64 + 2 * 32 * nd)


def test_backward_kernels_do_not_grow_with_the_observation():
    """Only the forward cell kernel stages the gathered inputs; the reverse cell step and the weight-gradient GEMM
    (which walks the encoder inputs in 64-column tiles) use a fixed amount whatever n_s is."""
    assert bwd_smem_bytes(4) == 99328 and bwd_smem_bytes(2) == 82944
    assert max(wgrad_smem_bytes(nd) for nd in (16, 32, 64, 128, 256)) == 81920
    assert max(bwd_smem_bytes(4), wgrad_smem_bytes(256)) <= SMEM_LIMIT


# widest own-observation width n_s whose FFMA cell kernel fits 227 KB, by neighbour count 0..4 (n_a = 4, n_h = 64).
# Worked out from fwd_smem_floats: the kernel needs 64 * ld_in + 64 * (s_dim + 68) + 2048 floats <= 58 112, i.e.
# ld_in <= 744 (s_dim = 64) or 616 (NeurComm cell, s_dim = 192), with ld_in = up4(K) + up4(n_a * nbr) + 64 * nbr
# (CommNet: + 64 once; IA2C: the observation alone).
WIDEST = {'ia2c': [744, 372, 248, 186, 148], 'ma2c_cu': [744, 744, 744, 744, 744],
          'ma2c_ic3': [None, 340, 226, 170, 136], 'ma2c_dial': [744, 340, 205, 138, 97],
          'ma2c_nc': [616, 274, 160, 103, 68], 'ia2c_fp': [616, 274, 160, 103, 68]}


def _full(variant, k, n_s, n_a=4):
    """k + 1 fully connected agents: every agent has exactly k neighbours"""
    from deeprl_network_b200.layout import ModelLayout
    from gpu_common import widths
    mask = 1 - np.eye(k + 1, dtype=int)
    return ModelLayout(variant, widths(variant, mask, n_s, n_a), n_a, mask)


@pytest.mark.parametrize('variant', list(WIDEST))
def test_widest_observation_that_fits_shared_memory(variant):
    from deeprl_network_b200 import layout as LY
    assert LY.SMEM_LIMIT == SMEM_LIMIT
    s_dim = 3 * NH if variant in ('ma2c_nc', 'ia2c_fp') else NH
    for k, n_s in enumerate(WIDEST[variant]):
        if n_s is None:                    # CommNet has no agent without neighbours
            continue
        lay = _full(variant, k, n_s)
        assert LY.ffma_fwd_smem_bytes(lay.ld_in, lay.s_dim, lay.n_h) == fwd_smem_bytes(lay.ld_in, s_dim) <= SMEM_LIMIT
        with pytest.raises(ValueError, match='limit is %d B' % SMEM_LIMIT):
            _full(variant, k, n_s + 1)
        # the paper value is the formula's: one more observation column does not fit
        ld = lambda w: up4(w if variant == 'ma2c_cu' else w * (1 + k)) + lay.kp_pad + lay.km_pad
        assert fwd_smem_bytes(ld(n_s), s_dim) <= SMEM_LIMIT < fwd_smem_bytes(ld(n_s + 1), s_dim)


def test_narrow_lstm_widths_share_the_limit():
    from deeprl_network_b200 import layout as LY
    from deeprl_network_b200.layout import ModelLayout
    mask = mask_of('chain8')
    for H in (16, 32):
        lay = ModelLayout('ma2c_nc', [5] * 8, 4, mask, n_h=H, n_fc=H)
        assert LY.ffma_fwd_smem_bytes(lay.ld_in, lay.s_dim, H) == fwd_smem_bytes(lay.ld_in, 3 * H, H=H) < SMEM_LIMIT
