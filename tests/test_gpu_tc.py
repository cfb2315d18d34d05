"""GPU: the wgmma tensor-core building blocks.  3xTF32 split GEMM with both operands in 128B-swizzled shared
memory (B via bulk copies), FP32 accumulation in registers, against float64."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


# every wgmma width the kernels use (m64n64k8 ... m64n256k8), K from one 8-deep k-step to several 32-deep k-blocks,
# with K % 32 != 0 (a partial last k-block) at every width
@pytest.mark.parametrize('M,K,N', [(128, 32, 256), (256, 256, 256), (128, 8, 64), (128, 16, 64), (384, 128, 64), (128, 72, 256),
                                   (128, 8, 128), (256, 40, 128), (128, 256, 128), (384, 104, 128),
                                   (128, 8, 192), (256, 56, 192), (128, 256, 192), (384, 136, 192),
                                   (256, 200, 64), (256, 24, 256)])
def test_3xtf32_gemm_matches_fp64(M, K, N):
    from deeprl_network_b200 import _lib as L
    lib = L.lib()
    lib.nmarl_tc_gemm_selftest.argtypes = [C.c_void_p] * 3 + [C.c_int] * 3 + [C.c_void_p] * 3
    rs = np.random.RandomState(0)
    A = (rs.randn(M, K) * np.exp(rs.randn(M, K))).astype(np.float32)          # wide dynamic range
    W = (rs.randn(K, N) / np.sqrt(K)).astype(np.float32)
    a, w = torch.tensor(A).cuda(), torch.tensor(W).cuda()
    c = torch.full((M, N), float('nan'), device='cuda')
    scratch = torch.zeros(((K + 31) // 32) * 2 * N * 32, device='cuda')
    err = torch.zeros(1, dtype=torch.int32, device='cuda')
    L.check(lib.nmarl_tc_gemm_selftest(a.data_ptr(), w.data_ptr(), c.data_ptr(), M, K, N, scratch.data_ptr(), err.data_ptr(),
                                       L.stream()), 'tc selftest')
    torch.cuda.synchronize()
    assert int(err.item()) == 0, 'pipeline timeout code %d' % int(err.item())
    ref = A.astype(np.float64) @ W.astype(np.float64)
    got = c.cpu().numpy().astype(np.float64)
    scale = np.abs(A).astype(np.float64) @ np.abs(W).astype(np.float64)        # sum |a||b| bounds the round-off
    rel = np.abs(got - ref) / scale
    assert np.isfinite(got).all()
    assert rel.max() < 2e-6, rel.max()                 # ~fp32 accuracy (plain TF32 would be ~5e-4)
    fp32 = (a @ w).cpu().numpy().astype(np.float64)
    assert np.abs(got - ref).max() <= 4 * np.abs(fp32 - ref).max() + 1e-6 * scale.max()


@pytest.mark.parametrize('variant', ['ma2c_nc', 'ma2c_ic3', 'ma2c_dial', 'ia2c'])
def test_tensor_core_cell_matches_ffma_cell(variant):
    """The tensor-core forward (B % 128 == 0) and the FP32-FFMA forward are two implementations of the same
    step: identical pi / v / state to ~1e-6, identical sampled actions, DIAL messages included."""
    import sys, os
    sys.path.insert(0, os.path.dirname(__file__))
    from gpu_common import bn, make_pair, nb, obs_dev, to_dev
    from deeprl_network_b200 import _lib as L
    from deeprl_network_b200.agents.engine import PolicyEngine
    B = 384
    eng, orc, lay, params = make_pair(variant, B)
    assert eng.use_tc
    ref = PolicyEngine(lay, B, 4, eng.hp, flat_params=lay.pack(params), use_tc=False)
    rs = np.random.RandomState(1)
    base = rs.randn(B, 8, 5).astype(np.float32); fp = rs.dirichlet(np.ones(4), size=(B, 8)).astype(np.float32)
    done = (rs.rand(B) < 0.3).astype(np.float32)
    c0 = (rs.randn(B, 8, 64) * .5).astype(np.float32); h0 = (rs.rand(B, 8, 64) - .5).astype(np.float32)
    u = to_dev(rs.rand(8, B), torch.float64)
    outs = []
    for e in (eng, ref):
        e.set_states(nb(c0), nb(h0))
        pi = torch.zeros(8, B, 4, device='cuda'); act = torch.zeros(8, B, dtype=torch.int32, device='cuda'); v = torch.zeros(8, B, device='cuda')
        e.step_p(obs_dev(lay, base), nb(fp), to_dev(done), pi, act, L.SAMPLE_UNIFORM, uniforms=u)
        e.step_v(obs_dev(lay, base), nb(fp), to_dev(done), act, v)
        e.check_tc()
        outs.append((pi, act, v, e.get_states_fw().clone(), None if e.msg[e.cur] is None else e.msg[e.cur].clone()))
    torch.testing.assert_close(outs[0][0], outs[1][0], rtol=0, atol=4e-6)
    torch.testing.assert_close(outs[0][2], outs[1][2], rtol=0, atol=5e-6)
    torch.testing.assert_close(outs[0][3], outs[1][3], rtol=0, atol=4e-6)
    assert (outs[0][1] != outs[1][1]).float().mean().item() < 0.002          # only at cdf boundaries
    if outs[0][4] is not None:
        torch.testing.assert_close(outs[0][4], outs[1][4], rtol=0, atol=4e-6)
