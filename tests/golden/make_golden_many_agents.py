"""Generate the many-agent CACC fixtures (N = 61 and N = 128 vehicles) by running the UNMODIFIED reference env.

Run in the authoring container only (needs the reference checkout, see make_golden.REF):
    python tests/golden/make_golden_many_agents.py [--force]
Writes tests/golden/many{61,128}_*.npz.  The fixtures are committed; nothing at test or bench time reads the reference.

Each case is make_golden.env_case(..., n_vehicle=N) on a shipped reference config.  N = 61 runs the tail of np.sum's
pairwise block (61 is not a multiple of 8), N = 128 the largest block NumPy sums without recursing.  The cases cover:
  * catchup_rand   catch-up, train mode, global reward (coop_gamma = -1), random actions
  * slowdown_test  slow-down, test mode, spatial reward (coop_gamma = 0.8), random actions
  * slowdown_crash slow-down, train mode, global reward, no control (const0): the platoon collides at step 107; with
                   batch_size = 10 the episode ends at step 110, so the frozen -G steps and the done flag are recorded
To keep each file under about 1 MB the two collision-free episodes keep their first STEPS steps, and every episode keeps
the headways of each step but only the last speeds / accelerations (`vs_last`, `us_last`).  `u01` is the uniform the
reference's reset drew (np.random.seed(seed); np.random.rand()), so a batched device env can be reset to the same
initial condition.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

STEPS = 60
CASES = [('catchup_rand', 'config_ma2c_nc_catchup.ini', 'rand', {}),
         ('slowdown_test', 'config_ma2c_cnet_slowdown.ini', 'rand', dict(test_mode=True, coop_gamma=0.8)),
         ('slowdown_crash', 'config_ma2c_cnet_slowdown.ini', 'const0', dict(batch_size=10))]


def many_case(CACCEnv, n, ini, kind, test_mode=False, **over):
    full = mg.env_case(CACCEnv, ini, kind, test_mode=test_mode, n_vehicle=n, **over)
    seed = int(full['ep0_seed_after']) - (2 if test_mode else 1)      # the seed the recorded reset used
    np.random.seed(seed)
    u01 = np.random.rand()
    steps = len(full['ep0_done'])
    keep = steps if full['ep0_done'][-1] and steps < 2 * STEPS else STEPS
    out = {k: full[k] for k in ('n_ep', 'ini', 'kind', 'test_mode', 'over', 'ep0_h0', 'ep0_v0', 'ep0_seed_after', 'ep0_v0s')}
    for k in ('acts', 'rew', 'done', 'greward', 'hs'):
        out['ep0_' + k] = full['ep0_' + k][:keep]
    out['ep0_obs'] = full['ep0_obs'][:keep + 1]
    out['ep0_vs_last'] = full['ep0_vs'][keep - 1]
    out['ep0_us_last'] = full['ep0_us'][keep - 1]
    out['ep0_u01'] = np.float64(u01)
    out['n_vehicle'] = n
    return out


def main():
    CACCEnv, _ = mg._import_reference()
    for n in (61, 128):
        for name, ini, kind, kw in CASES:
            path = os.path.join(HERE, 'many%d_%s.npz' % (n, name))
            if os.path.exists(path) and '--force' not in sys.argv:
                continue
            out = many_case(CACCEnv, n, ini, kind, **kw)
            np.savez_compressed(path, **out)
            print(os.path.basename(path), 'steps', len(out['ep0_done']), 'done', bool(out['ep0_done'][-1]),
                  'sumG', float(np.sum(out['ep0_greward'])), 'bytes', os.path.getsize(path))


if __name__ == '__main__':
    main()
