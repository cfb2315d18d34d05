"""GPU: K8-K10 -- training forward, A2C loss, BPTT through the message graph, weight gradients,
global-norm clip and TF-semantics RMSProp -- against oracle autograd (fp64 oracle bounds the error)."""
import numpy as np
import pytest
import torch

from gpu_common import HP, bn, make_pair, nb, obs_dev, oracle_obs, to_dev

pytestmark = pytest.mark.gpu
VARIANTS = ['ma2c_nc', 'ma2c_ic3', 'ma2c_dial', 'ia2c', 'ia2c_fp', 'ma2c_cu']


def _batch(eng, lay, T, B, seed=0, N=8, n_s=5, n_a=4, poison=False):
    """Draw a training batch and load it into the engine's buffers.  poison: NaN in the padding columns of obs_buf."""
    rs = np.random.RandomState(seed)
    base = rs.randn(T, B, N, n_s).astype(np.float32)
    fp = rs.dirichlet(np.ones(n_a), size=(T, B, N)).astype(np.float32)
    acts = rs.randint(0, n_a, size=(T, B, N))
    dones = np.zeros((T, B), dtype=np.float32); dones[0, ::2] = 1
    if T > 3:
        dones[3, 0] = 1
    Rs = rs.randn(T, B, N).astype(np.float32); Advs = rs.randn(T, B, N).astype(np.float32)
    c0 = (rs.randn(B, N, 64) * .5).astype(np.float32); h0 = (rs.rand(B, N, 64) - .5).astype(np.float32)
    eng.T_cur = T
    for t in range(T):
        eng.obs_buf[t].copy_(obs_dev(lay, base[t], poison=poison))
    eng.fp_buf[:T].copy_(to_dev(np.transpose(fp, (0, 2, 1, 3))))
    eng.act_buf[:T].copy_(to_dev(np.transpose(acts, (0, 2, 1)), torch.int32))
    eng.done_buf[:T].copy_(to_dev(dones))
    eng.Rs[:T].copy_(to_dev(np.transpose(Rs, (0, 2, 1)))); eng.Advs[:T].copy_(to_dev(np.transpose(Advs, (0, 2, 1))))
    eng.set_states(nb(c0), nb(h0))
    return base, fp, acts, dones, Rs, Advs, c0, h0


def _oracle_backward(orc, lay, batch, lr=5e-4, apply=False, hp=HP):
    base, fp, acts, dones, Rs, Advs, c0, h0 = batch
    T = len(base)
    st = torch.tensor(np.concatenate([c0, h0], -1), dtype=orc.dtype)
    orc.states_bw = st.clone(); orc.states_fw = st.clone()
    obs_t = [oracle_obs(lay, base[t]) for t in range(T)]
    return orc.backward(obs_t, fp, acts, dones, Rs, Advs, lr, v_coef=hp['v_coef'], e_coef=hp['e_coef'],
                        max_grad_norm=hp['max_grad_norm'], alpha=hp['alpha'], epsilon=hp['epsilon'], apply=apply)


@pytest.mark.parametrize('variant', VARIANTS)
@pytest.mark.parametrize('T,B', [(6, 1), (5, 37), (3, 130), (3, 128), (4, 256)])    # B % 128 == 0: tensor-core forward + backward
def test_gradients_match_oracle_autograd(variant, T, B):
    eng, orc, lay, params = make_pair(variant, B, T=T, dtype=torch.float64)
    batch = _batch(eng, lay, T, B)
    summ = _oracle_backward(orc, lay, batch)
    eng.backward()
    torch.cuda.synchronize()
    eng.check_tc()
    g = lay.unpack(eng.grads.cpu().numpy())
    worst = 0.0
    for name in orc.names:
        ref = orc.grads[name].numpy()
        err = np.abs(g[name] - ref).max()
        scale = max(1e-3, np.abs(ref).max())
        worst = max(worst, err / scale)
        assert err <= 2e-5 * scale + 1e-7, (name, err, scale)
    # loss terms (per agent)
    ls = eng.losses()
    np.testing.assert_allclose(ls['policy_loss'], summ['policy_loss'], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(ls['value_loss'], summ['value_loss'], rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(ls['entropy_loss'], summ['entropy_loss'], rtol=1e-4, atol=1e-5)
    # training-forward pi/v are visible through the saved head gradients only; check the saved states instead
    pad = np.ones(lay.n_param, bool)
    for _, o, s in lay.entries:
        pad[o:o + int(np.prod(s))] = False
    assert np.all(eng.grads.cpu().numpy()[pad] == 0)          # alignment padding never receives gradient


@pytest.mark.parametrize('variant', VARIANTS)
def test_clip_and_rmsprop_step(variant):
    hp = dict(HP, max_grad_norm=0.05)                          # make the clip active
    T, B = 4, 9
    eng, orc, lay, params = make_pair(variant, B, T=T, hp=hp)
    batch = _batch(eng, lay, T, B, seed=4)
    for it in range(2):                                         # second step exercises ms != 1
        summ = _oracle_backward(orc, lay, batch, lr=1e-2, apply=True, hp=hp)
        eng.set_states(nb(batch[6]), nb(batch[7]))
        eng.backward(); eng.apply(1e-2)
        torch.cuda.synchronize()
        np.testing.assert_allclose(eng.norm_out.cpu().numpy(), summ['grad_norm'], rtol=2e-4)
        w = lay.unpack(eng.params.cpu().numpy())
        for name in orc.names:
            np.testing.assert_allclose(w[name], orc.p[name].detach().numpy(), rtol=0, atol=3e-6, err_msg=name)
    assert np.array(summ['grad_norm']).min() > 0.05
    # states_bw := states_fw after the update (policies.py:211)
    assert torch.equal(eng.h_bw, eng.h[eng.cur]) and torch.equal(eng.c_bw, eng.c[eng.cur])


def test_sharded_gradients_add_up():
    """Data-parallel identity used by the multi-GPU path: with the loss scaled by 1/(T*B_total),
    the SUM of per-shard gradients equals the single-process gradient (clip AFTER the reduce)."""
    T, B = 4, 12
    eng, orc, lay, params = make_pair('ma2c_nc', B, T=T)
    batch = _batch(eng, lay, T, B, seed=7)
    eng.backward()
    full = eng.grads.clone()
    total = torch.zeros_like(full)
    for lo, hi in ((0, 5), (5, 12)):
        sub, _, _, _ = make_pair('ma2c_nc', hi - lo, T=T)
        sub.world = 1
        sb = tuple(x[:, lo:hi] if x.ndim >= 2 and x.shape[0] == T else x[lo:hi] for x in batch)
        sub.T_cur = T
        sub.obs_buf[:T, :, :, :5].copy_(to_dev(np.transpose(sb[0], (0, 2, 1, 3))))
        sub.fp_buf[:T].copy_(to_dev(np.transpose(sb[1], (0, 2, 1, 3))))
        sub.act_buf[:T].copy_(to_dev(np.transpose(sb[2], (0, 2, 1)), torch.int32))
        sub.done_buf[:T].copy_(to_dev(sb[3]))
        sub.Rs[:T].copy_(to_dev(np.transpose(sb[4], (0, 2, 1)))); sub.Advs[:T].copy_(to_dev(np.transpose(sb[5], (0, 2, 1))))
        sub.set_states(nb(sb[6]), nb(sb[7]))
        a = sub._bwd_args(T)
        a.B_total = B                                          # what world_size > 1 sets
        sub.h_seq[0].copy_(sub.h_bw); sub.c_seq[0].copy_(sub.c_bw)
        from deeprl_network_b200 import _lib as L
        import ctypes as C
        L.check(L.lib().nmarl_a2c_backward(C.byref(sub.model), C.byref(a), L.stream()), 'bwd')
        total += sub.grads
    torch.testing.assert_close(total, full, rtol=1e-4, atol=1e-7)
