"""CPU: the data layouts of the tensor-core path, checked without a GPU.

* The LSTM state layout follows from the path: feature-major on tensor cores except for DIAL, env-major elsewhere.
  nmarl_policy_step_p / _v and nmarl_a2c_bptt refuse a call whose state_fm declares the other layout, before any
  CUDA call (dummy non-null pointers, never dereferenced).
* The weight-gradient operand tiles sv_dzT / sv_dpT: every float range tc_cell_bwd_kernel writes (one raw tile per
  step, agent and 32-env block) and every range tc_wgrad_kernel bulk-copies, both enumerated through
  nmarl_operand_tile_offset as the kernels address them, cover the engine's allocation exactly, without gaps.
"""
import ctypes

import numpy as np
import pytest

from deeprl_network_b200 import _lib as L
from deeprl_network_b200.agents.engine import operand_tile_shapes, tc_eligible
from deeprl_network_b200.envs.cacc_env import chain_masks
from deeprl_network_b200.layout import ModelLayout

NH = 64
RULE = b'state_fm must be 1 on the tensor-core path except for DIAL, else 0'


def _layout(variant, N=8):
    mask = chain_masks(N)[0]
    n_s = [5 * (1 + int(mask[i].sum())) for i in range(N)] if variant == 'ia2c' else [5] * N
    return ModelLayout(variant, n_s, 4, mask, obs_mode='gather')


def _fill(args, B, state_fm):
    """every pointer a distinct dummy (never dereferenced: the refusal comes first), sizes for B envs"""
    for k, (name, ty) in enumerate(type(args)._fields_):
        if ty is ctypes.c_void_p:
            setattr(args, name, 4096 + 256 * k)
    args.B, args.state_fm = B, state_fm
    return args


def _calls(lay, B, state_fm):
    lib = L.lib()
    m = lay.c_model()
    f = _fill(L.FwdArgs(), B, state_fm)
    f.sample_mode = L.SAMPLE_NONE
    b = _fill(L.BwdArgs(), B, state_fm)
    b.T, b.B_total = 2, B
    return {'policy_step_p': lambda: lib.nmarl_policy_step_p(ctypes.byref(m), ctypes.byref(f), None),
            'policy_step_v': lambda: lib.nmarl_policy_step_v(ctypes.byref(m), ctypes.byref(f), None),
            'a2c_backward': lambda: lib.nmarl_a2c_bptt(ctypes.byref(m), ctypes.byref(b), None)}


@pytest.mark.parametrize('variant,B,state_fm', [
    ('ma2c_nc', 128, 0), ('ma2c_ic3', 128, 0), ('ia2c', 128, 0),        # tensor cores: feature-major required
    ('ma2c_dial', 128, 1),                                               # DIAL: env-major on tensor cores too
    ('ma2c_nc', 96, 1),                                                  # FFMA path (B % 128 != 0): env-major
])
def test_calls_refuse_the_other_state_layout(variant, B, state_fm):
    lay = _layout(variant)
    assert tc_eligible(lay, B) == (B % 128 == 0)
    for name, call in _calls(lay, B, state_fm).items():
        assert call() != 0, name
        err = L.lib().nmarl_last_error()
        assert err.startswith(name.encode() + b': ') and RULE in err and err.endswith(b'(got %d)' % state_fm), err


# ---- operand tiles --------------------------------------------------------------------------------------------------
def _wgrad_splits(n_agent):
    """nmarl_tc_wgrad_splits (tc_wgrad.cu)"""
    s = 33
    while 4 * s * n_agent > 132 * 8 and s > 1:
        s = (s + 1) // 2
    return s


def _merge(iv):
    """union of [start, end) float ranges as a sorted list of disjoint ranges"""
    out = []
    for s, e in sorted(iv):
        if out and s <= out[-1][1]:
            out[-1][1] = max(out[-1][1], e)
        else:
            out.append([s, e])
    return out


def _written(off, variant, rows, N, B, T, dz):
    """tc_cell_bwd_kernel: reverse step t writes through the step base train.cu passes (tile (t, 0, 0)); CTA
    (x, agent i), warp half rh writes the tile of block 2 x + rh, tile rows: dz^T every gate column, dpre^T the
    encoder pre-activation columns put_dp stores"""
    if dz:
        cols = {g * NH + u for g in range(4) for u in range(NH)}
    elif variant in ('ma2c_nc', 'ia2c'):
        cols = {gp * NH + u for gp in range({'ma2c_nc': 3, 'ia2c': 1}[variant]) for u in range(NH)}
    else:
        cols = {u for u in range(2 * NH)}
    assert cols == set(range(rows)), 'every row of the tile is written'
    iv = []
    for t in range(T):
        base = off(rows, t, N, B, 0, 0)
        for i in range(N):
            for x in range(B // 64):
                for rh in range(2):
                    s = base + off(rows, 0, N, B, i, 2 * x + rh)
                    iv.append((s, s + rows * 32))
    return iv


def _read(off, lay, variant, rows, N, B, T, dz):
    """tc_wgrad_kernel: per (split, job, agent) the issuer bulk-copies rows [n_row0, n_row0 + N_job) of the tile of
    every k-block (t, rb) of its split (job_desc, fetch)"""
    if dz:
        jobs = [(0, 256)] * (2 if lay.s_dim + NH > 128 else 1)
    else:
        jobs = [(0, rows)]
        if variant != 'ia2c':
            jobs += [(128 if variant == 'ma2c_nc' else 64, 64)] * (2 if lay.km_pad > 128 else 1)
    bpt = B // 32
    total, splits = T * bpt, _wgrad_splits(N)
    per = -(-total // splits)
    iv = []
    for n_row0, n_job in jobs:
        for sp in range(splits):
            for i in range(N):
                for kb in range(sp * per, min(total, sp * per + per)):
                    s = off(rows, kb // bpt, N, B, i, kb % bpt) + n_row0 * 32
                    iv.append((s, s + n_job * 32))
    return iv


@pytest.mark.parametrize('variant,N,B,T', [('ma2c_nc', 8, 4096, 60),             # the headline workload
                                           ('ma2c_nc', 8, 128, 8), ('ma2c_ic3', 8, 128, 8),
                                           ('ma2c_dial', 8, 128, 8), ('ia2c', 8, 128, 8)])
def test_operand_tiles_written_and_read_cover_the_allocation(variant, N, B, T):
    off = L.lib().nmarl_operand_tile_offset
    lay = _layout(variant, N)
    assert tc_eligible(lay, B)
    shapes = operand_tile_shapes(variant, N, B, T, NH)
    ndp = {'ma2c_nc': 3 * NH, 'ia2c': NH}.get(variant, 2 * NH)
    for dz, rows, shape in ((True, 4 * NH, shapes[0]), (False, ndp, shapes[1])):
        alloc = int(np.prod(shape))
        # the [hi | lo] pair layout this replaced allocated two tiles per 32 env rows
        assert 2 * alloc == T * N * (B // 32) * 2 * rows * 32
        w = _merge(_written(off, variant, rows, N, B, T, dz))
        r = _merge(_read(off, lay, variant, rows, N, B, T, dz))
        assert w == r, (variant, dz, 'the wgrad kernel reads exactly what the backward cell kernel writes')
        assert w == [[0, alloc]], (variant, dz, 'the tiles fill the allocation without gaps or overrun')
