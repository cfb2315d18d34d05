"""Generate the heterogeneous IA2C / IA2C_FP / IA2C_CU fixtures by running the UNMODIFIED reference code on the TF shim.

Run in the authoring container only (needs the reference checkout, see make_golden.REF):
    python tests/golden/make_golden_hetero_ia2c.py [--force]
Writes tests/golden/hetero_{,iso_,iso0_}{ia2c,ia2c_fp,ma2c_cu}.npz.  The fixtures are committed; nothing at test or
bench time reads the reference.

Same agents, graphs, scripted stream and file format as make_golden.hetero_case (the MA2C-family fixtures): 6 agents
with n_s = [5,7,4,6,5,3], n_a = [4,3,5,2,4,3], 3 updates of 8 steps, the trained weights kept as a W1_SAMPLE sample.
What differs is how the agent classes are driven:
  * IA2C / IA2C_FP (agents/models.py:118-132, 171-188) are called with per-agent neighbour actions
    (forward(ob, done) / forward(ob, done, nactions, 'v') / add_transition(ob, nactions, ...)); an IA2C_FP agent sees
    its random observation with the neighbours' previous policies appended, as the environment would append them
    (envs/cacc_env.py:74-77).  `obs` holds the random observations only.
  * IA2C_CU (agents/models.py:261-275) has the MA2C signatures.
"""
import hashlib
import importlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

AGENTS = ('ia2c', 'ia2c_fp', 'ma2c_cu')


def hetero_ia2c_case(agent, edges, w1_sample=mg.W1_SAMPLE):
    sys.setrecursionlimit(100000)
    tf = importlib.import_module('tf_shim')
    sys.modules['tensorflow'] = tf
    for mod in ('agents.models', 'agents.policies', 'agents.utils', 'utils', 'envs.cacc_env'):
        sys.modules.pop(mod, None)
    import agents.models as am
    H = mg.HETERO
    N = len(H['n_s_ls'])
    mask = np.zeros((N, N), dtype=int)
    for a, b in edges:
        mask[a, b] = mask[b, a] = 1
    dist = np.zeros((N, N), dtype=int)
    mc = mg._cfg('config_ma2c_nc_catchup.ini')['MODEL_CONFIG']
    mc['batch_size'] = str(H['n_step'])
    cls = {'ia2c': am.IA2C, 'ia2c_fp': am.IA2C_FP, 'ma2c_cu': am.IA2C_CU}[agent]
    np.random.seed(12)
    model = cls(H['n_s_ls'], H['n_a_ls'], mask, dist, -1.0, 10 ** 6, mc, seed=12)
    assert not model.identical_agent
    w0 = tf.variable_values()
    rs = np.random.RandomState(3)
    T = H['n_step']
    log, obs_l, uni_l, rew_l = [], [], [], []
    fp = [np.ones(n) / n for n in H['n_a_ls']]
    done = True
    model.reset()
    nbr = [list(np.where(mask[i] == 1)[0]) for i in range(N)]
    indep = agent != 'ma2c_cu'

    def full_ob(ob, fp):
        if agent != 'ia2c_fp':
            return ob
        return [np.concatenate([ob[i]] + [np.asarray(fp[j], dtype=np.float64) for j in nbr[i]]) for i in range(N)]

    def nactions(act):
        return [act[nbr[i]] for i in range(N)]

    def observe():
        ob = [rs.randn(n) for n in H['n_s_ls']]
        obs_l.append(np.concatenate(ob))
        return ob

    def decide(ob, done, fp):
        pi = model.forward(full_ob(ob, fp), done) if indep else model.forward(ob, done, fp)
        pi = [np.asarray(p, dtype=np.float64).ravel() for p in pi]
        log.append(np.concatenate(pi))
        u = rs.rand(N)
        uni_l.append(u)
        act = []
        for i in range(N):
            cdf = np.cumsum(pi[i]); cdf = cdf / cdf[-1]
            act.append(int(np.searchsorted(cdf, u[i], side='right')))
        return pi, np.array(act)

    def value(ob, done, fp, act):
        if indep:
            return model.forward(full_ob(ob, fp), done, nactions(act), 'v')
        return model.forward(ob, done, fp, act, 'v')
    for upd in range(H['updates']):
        for t in range(T):
            ob = observe()
            pi, act = decide(ob, done, fp)
            v = value(ob, done, fp, act)
            log.append(np.asarray(v, dtype=np.float64).ravel())
            r = float(rs.randn() * 300.0)
            rew_l.append(r)
            if indep:
                model.add_transition(full_ob(ob, fp), nactions(act), act, r, v, False)
            else:
                model.add_transition(ob, fp, act, r, v, False)
            fp = [np.asarray(p, dtype=np.float32) for p in pi]
            done = False
        ob = observe()
        pi, act = decide(ob, done, fp)
        R = value(ob, done, fp, act)
        log.append(np.asarray(R, dtype=np.float64).ravel())
        model.backward(R, 0)
    w1 = tf.variable_values()
    out = dict(trace=np.concatenate(log), obs=np.concatenate(obs_l), uniforms=np.array(uni_l), rewards=np.array(rew_l),
               names=np.array(list(w0)), mask=mask, n_s_ls=np.array(H['n_s_ls']), n_a_ls=np.array(H['n_a_ls']),
               n_step=T, updates=H['updates'])
    for n in w0:
        out['w0sha/' + n] = hashlib.sha256(np.ascontiguousarray(w0[n]).tobytes()).hexdigest()
        out['w0shape/' + n] = np.array(w0[n].shape)
        if w1[n].size <= w1_sample:
            out['w1/' + n] = w1[n]
        else:
            idx = np.sort(np.random.RandomState(len(out)).choice(w1[n].size, w1_sample, replace=False)).astype(np.int32)
            out['w1idx/' + n] = idx
            out['w1/' + n] = np.ascontiguousarray(w1[n]).ravel()[idx]
    return out


def main():
    mg._import_reference()
    for prefix, edges in [('hetero_', mg.HETERO['edges'])] + list(mg.HETERO_ISO.items()):
        for agent in AGENTS:
            name = prefix + agent
            if os.path.exists(os.path.join(HERE, name + '.npz')) and '--force' not in sys.argv:
                continue
            out = hetero_ia2c_case(agent, edges)
            np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
            print(name, 'trace', out['trace'].shape, 'n_var', len(out['names']))


if __name__ == '__main__':
    main()
