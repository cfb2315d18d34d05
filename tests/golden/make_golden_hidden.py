"""Generate the LSTM-width fixtures (num_lstm = num_fc = 16 / 32) by running the UNMODIFIED reference code on the TF shim.

Run in the authoring container only (needs the reference checkout, see make_golden.REF):
    python tests/golden/make_golden_hidden.py [--force]
Writes tests/golden/tfnet_h{16,32}_<agent>.npz and tests/golden/hetero_h32_{ma2c_nc,ia2c_fp}.npz.  The fixtures are
committed; nothing at test or bench time reads the reference.

  * tfnet_h*: make_golden.tfnet_case -- the reference env + Trainer + agent class on one of the six `config/*` files,
    100 training steps -- with MODEL_CONFIG num_lstm = num_fc = the width.  Everything else is the shipped config.
  * hetero_h32_*: make_golden.hetero_case (NeurComm) and make_golden_hetero_ia2c.hetero_ia2c_case (IA2C_FP) on the
    graph whose last agent has no neighbour (make_golden.HETERO_ISO['hetero_iso_']), at width 32.
The case functions are used unchanged; only the MODEL_CONFIG they read is overridden.  `n_h` records the width.  The
trained weights are kept as a W1_SAMPLE sample per tensor ('w1idx/<name>' = flat indices, 'w1/<name>' = the values),
as in the heterogeneous fixtures; the pi / v / R trace stays complete.  Each case runs in a fresh process so that the
shim's variable registry starts empty.
"""
import multiprocessing as mp
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

TFNET = [('ma2c_nc', 'config_ma2c_nc_catchup.ini'), ('ia2c', 'config_ia2c_slowdown.ini'),
         ('ia2c_fp', 'config_ia2c_fp_catchup.ini'), ('ma2c_ic3', 'config_ma2c_cnet_slowdown.ini'),
         ('ma2c_dial', 'config_ma2c_dial_catchup.ini'), ('ma2c_cu', 'config_ia2c_cu_catchup.ini')]
WIDTHS = (16, 32)
TOTAL_STEP = 100
HETERO_WIDTH = 32


def _with_width(n_h):
    """make_golden._cfg with MODEL_CONFIG num_lstm = num_fc = n_h"""
    base = mg._cfg

    def cfg(name, **over):
        cp = base(name, **over)
        cp['MODEL_CONFIG']['num_lstm'] = str(n_h)
        cp['MODEL_CONFIG']['num_fc'] = str(n_h)
        return cp
    mg._cfg = cfg


def _sample_w1(out):
    """trained weights -> W1_SAMPLE entries per tensor (make_golden.hetero_case's recipe)"""
    for n in [str(x) for x in out['names']]:
        w = out.pop('w1/' + n)
        out['w0shape/' + n] = np.array(w.shape)
        if w.size <= mg.W1_SAMPLE:
            out['w1/' + n] = w
        else:
            idx = np.sort(np.random.RandomState(len(out)).choice(w.size, mg.W1_SAMPLE, replace=False)).astype(np.int32)
            out['w1idx/' + n] = idx
            out['w1/' + n] = np.ascontiguousarray(w).ravel()[idx]
    return out


def run_case(job):
    kind, agent, ini, n_h, name = job
    mg._import_reference()
    _with_width(n_h)
    if kind == 'tfnet':
        out = _sample_w1(mg.tfnet_case(ini, TOTAL_STEP))
    elif agent == 'ma2c_nc':
        out = mg.hetero_case(agent, mg.HETERO_ISO['hetero_iso_'], w1_sample=mg.W1_SAMPLE)
    else:
        import make_golden_hetero_ia2c as mgi
        out = mgi.hetero_ia2c_case(agent, mg.HETERO_ISO['hetero_iso_'])
    out['n_h'] = n_h
    np.savez_compressed(os.path.join(HERE, name + '.npz'), **out)
    return name, out['trace'].shape, len(out['names'])


def main():
    jobs = [('tfnet', a, ini, h, 'tfnet_h%d_%s' % (h, a)) for h in WIDTHS for a, ini in TFNET]
    jobs += [('hetero', a, None, HETERO_WIDTH, 'hetero_h%d_%s' % (HETERO_WIDTH, a)) for a in ('ma2c_nc', 'ia2c_fp')]
    jobs = [j for j in jobs if '--force' in sys.argv or not os.path.exists(os.path.join(HERE, j[-1] + '.npz'))]
    with mp.get_context('spawn').Pool(min(len(jobs), os.cpu_count() or 1) or 1, maxtasksperchild=1) as pool:
        for name, shape, n_var in pool.imap_unordered(run_case, jobs):
            print(name, 'trace', shape, 'n_var', n_var, flush=True)


if __name__ == '__main__':
    main()
