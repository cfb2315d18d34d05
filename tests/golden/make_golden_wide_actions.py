"""Generate the wide-action fixtures (agents with 8 to 15 actions) by running the UNMODIFIED reference code on the TF shim.

Run in the authoring container only (needs the reference checkout, see make_golden.REF):
    python tests/golden/make_golden_wide_actions.py [--force]
Writes tests/golden/wide_{ma2c_nc,ma2c_dial,ia2c_fp}.npz, tests/golden/wide_iso_ia2c_fp.npz,
tests/golden/wide_n12_ma2c_nc.npz and tests/golden/wide_n12_h16_ma2c_nc.npz.  The fixtures are committed; nothing at test or bench time reads the reference.

  * wide_ma2c_nc / wide_ma2c_dial: make_golden.hetero_case on the HETERO graph.
  * wide_ia2c_fp: make_golden_hetero_ia2c.hetero_ia2c_case on the HETERO graph; wide_iso_ia2c_fp on the graph whose
    last agent has no neighbour (make_golden.HETERO_ISO['hetero_iso_']).
  * wide_n12_ma2c_nc: identical agents (every n_s = 5, every n_a = 12) on the HETERO graph, which takes the
    reference's `identical_agent` branch (agents/models.py:90-94, NCMultiAgentPolicy with lstm_comm) -- the
    homogeneous path the batched engine and the C ABI run.  make_golden.hetero_case refuses identical agents, so
    identical_case below drives the same scripted stream (same seeds, same recording) without that check.
  * wide_n12_h16_ma2c_nc: wide_n12_ma2c_nc at num_lstm = num_fc = 16 (make_golden_hidden's width override), the
    point where the narrow LSTM width meets the 16-wide head.  `n_h` records the width.
The case functions are used unchanged; only the action counts they read are overridden: n_a_ls = N_A_LS, which mixes
narrow agents with agents of 8 to 15 actions (the 16-wide head of the kernels).  The trained weights are kept as a
W1_SAMPLE sample per tensor, as in the other heterogeneous fixtures.  Each case runs in a fresh process so that the
shim's variable registry starts empty.
"""
import hashlib
import importlib
import multiprocessing as mp
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

N_A_LS = [8, 3, 15, 2, 11, 6]
N_A_SAME, N_S_SAME = 12, 5
JOBS = [('wide_ma2c_nc', 'ma2c_nc', 'hetero'), ('wide_ma2c_dial', 'ma2c_dial', 'hetero'),
        ('wide_ia2c_fp', 'ia2c_fp', 'hetero'), ('wide_iso_ia2c_fp', 'ia2c_fp', 'hetero_iso_'),
        ('wide_n12_ma2c_nc', 'ma2c_nc', 'same'), ('wide_n12_h16_ma2c_nc', 'ma2c_nc', 'same')]
WIDTH = {'wide_n12_h16_ma2c_nc': 16}          # num_lstm = num_fc of the cases that override the config's 64


def identical_case(agent, edges):
    """make_golden.hetero_case's scripted stream for IDENTICAL agents: every agent has n_s = N_S_SAME observations and
    n_a = N_A_SAME actions, so the unmodified reference model takes its identical_agent branch.  Same seeds, same
    observation / reward / uniform stream, same recording and W1_SAMPLE as hetero_case."""
    sys.setrecursionlimit(100000)
    tf = importlib.import_module('tf_shim')
    sys.modules['tensorflow'] = tf
    for mod in ('agents.models', 'agents.policies', 'agents.utils', 'utils', 'envs.cacc_env'):
        sys.modules.pop(mod, None)
    import agents.models as am
    H = mg.HETERO
    N = len(H['n_s_ls'])
    n_s_ls, n_a_ls = [N_S_SAME] * N, [N_A_SAME] * N
    mask = np.zeros((N, N), dtype=int)
    for a, b in edges:
        mask[a, b] = mask[b, a] = 1
    mc = mg._cfg('config_ma2c_nc_catchup.ini')['MODEL_CONFIG']
    mc['batch_size'] = str(H['n_step'])
    np.random.seed(12)
    model = {'ma2c_nc': am.MA2C_NC}[agent](n_s_ls, n_a_ls, mask, np.zeros((N, N), dtype=int), -1.0, 10 ** 6, mc, seed=12)
    assert model.identical_agent
    w0 = tf.variable_values()
    rs = np.random.RandomState(3)
    T = H['n_step']
    log, obs_l, uni_l, rew_l = [], [], [], []
    fp = [np.ones(n) / n for n in n_a_ls]
    done = True
    model.reset()

    def decide(ob, done, fp):
        pi = [np.asarray(p, dtype=np.float64).ravel() for p in model.forward(ob, done, fp)]
        log.append(np.concatenate(pi))
        u = rs.rand(N)
        uni_l.append(u)
        act = []
        for i in range(N):
            cdf = np.cumsum(pi[i]); cdf = cdf / cdf[-1]
            act.append(int(np.searchsorted(cdf, u[i], side='right')))
        return pi, np.array(act)
    for upd in range(H['updates']):
        for t in range(T):
            ob = [rs.randn(n) for n in n_s_ls]
            obs_l.append(np.concatenate(ob))
            pi, act = decide(ob, done, fp)
            v = model.forward(ob, done, fp, act, 'v')
            log.append(np.asarray(v, dtype=np.float64).ravel())
            r = float(rs.randn() * 300.0)
            rew_l.append(r)
            model.add_transition(ob, fp, act, r, v, False)
            fp = [np.asarray(p, dtype=np.float32) for p in pi]
            done = False
        ob = [rs.randn(n) for n in n_s_ls]
        obs_l.append(np.concatenate(ob))
        pi, act = decide(ob, done, fp)
        R = model.forward(ob, done, fp, act, 'v')
        log.append(np.asarray(R, dtype=np.float64).ravel())
        model.backward(R, 0)
    w1 = tf.variable_values()
    out = dict(trace=np.concatenate(log), obs=np.concatenate(obs_l), uniforms=np.array(uni_l), rewards=np.array(rew_l),
               names=np.array(list(w0)), mask=mask, n_s_ls=np.array(n_s_ls), n_a_ls=np.array(n_a_ls),
               n_step=T, updates=H['updates'])
    for n in w0:
        out['w0sha/' + n] = hashlib.sha256(np.ascontiguousarray(w0[n]).tobytes()).hexdigest()
        out['w0shape/' + n] = np.array(w0[n].shape)
        if w1[n].size <= mg.W1_SAMPLE:
            out['w1/' + n] = w1[n]
        else:
            idx = np.sort(np.random.RandomState(len(out)).choice(w1[n].size, mg.W1_SAMPLE, replace=False)).astype(np.int32)
            out['w1idx/' + n] = idx
            out['w1/' + n] = np.ascontiguousarray(w1[n]).ravel()[idx]
    return out


def run_case(job):
    name, agent, graph = job
    mg._import_reference()
    if name in WIDTH:
        import make_golden_hidden
        make_golden_hidden._with_width(WIDTH[name])
    mg.HETERO['n_a_ls'] = list(N_A_LS)
    edges = mg.HETERO_ISO.get(graph, mg.HETERO['edges'])
    if graph == 'same':
        out = identical_case(agent, mg.HETERO['edges'])
    elif agent.startswith('ma2c_'):
        out = mg.hetero_case(agent, edges, w1_sample=mg.W1_SAMPLE)
    else:
        import make_golden_hetero_ia2c as mgi
        out = mgi.hetero_ia2c_case(agent, edges)
    if name in WIDTH:
        out['n_h'] = WIDTH[name]
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
    return name, out['trace'].shape, len(out['names'])


def main():
    jobs = [j for j in JOBS if '--force' in sys.argv or not os.path.exists(os.path.join(HERE, j[0] + '.npz'))]
    if not jobs:
        return
    with mp.get_context('spawn').Pool(min(len(jobs), os.cpu_count() or 1), maxtasksperchild=1) as pool:
        for name, shape, n_var in pool.imap_unordered(run_case, jobs):
            print(name, 'trace', shape, 'n_var', n_var, flush=True)


if __name__ == '__main__':
    main()
