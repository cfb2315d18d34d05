"""Cost of resumable training (TRAIN_CONFIG.checkpoint_interval) at 4096 envs x 8 agents, NeurComm catch-up.

    python tools/bench_resume.py [--n-env 4096] [--updates 10] [--rounds 4] [--repeats 3]

1. Wall time of one snapshot (VecTrainer.snapshot: device -> host copies, then resume.save_snapshot: torch.save to a
   temporary directory, fsync and rename) and of one restore (resume.load_snapshot, VecTrainer.restore into a fresh
   trainer, device synchronise); the median of `repeats`.  Also the snapshot file's size.
2. Update time between snapshots against a run without the key: two trainers of the same config (replayed CUDA
   graphs, as main.py runs them), `rounds` alternating rounds of `updates` updates each, timed with a device
   synchronise; the `with` trainer takes a snapshot between rounds (outside the timed window).  Median of the
   per-round means.  No kernel and no launch of the update path depends on the key, so both should agree within
   the spread of two trainers built side by side.

Prints a header line with the GPU name and its power limit, then one JSON line per measurement.  Writes only to a
temporary directory, which it removes.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_agents import gpu_info  # noqa: E402


def _trainer(n_env):
    import main
    from deeprl_network_b200 import utils as U
    cfg = main.read_config(os.path.join(ROOT, 'config', 'config_ma2c_nc_catchup.ini'))
    cfg['ENV_CONFIG']['n_env'] = str(n_env)
    env = main.init_env(cfg['ENV_CONFIG'])
    model = main.init_agent(env, cfg['MODEL_CONFIG'], 10 ** 9, cfg.getint('ENV_CONFIG', 'seed'))
    loop = U.VecTrainer(env, model, graph=True)
    loop.start()
    return cfg, loop


def _timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main_():
    import torch
    from deeprl_network_b200 import resume as R
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--n-env', type=int, default=4096)
    ap.add_argument('--updates', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=4)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    print(json.dumps(gpu_info()), flush=True)
    cfg_path = os.path.join(ROOT, 'config', 'config_ma2c_nc_catchup.ini')
    text = open(cfg_path).read()
    _, plain = _trainer(args.n_env)
    _, keyed = _trainer(args.n_env)
    for loop in (plain, keyed):
        loop.update()                                   # warm-up and graph capture
    per = {'without': [], 'with': []}
    with tempfile.TemporaryDirectory() as tmp:
        save_s, load_s = [], []
        for r in range(args.rounds):
            for name, loop in (('without', plain), ('with', keyed)):
                dt, _ = _timed(lambda: [loop.update() for _ in range(args.updates)])
                per[name].append(dt / args.updates)
            # the snapshot itself, between rounds, outside the timed window
            dt, _ = _timed(lambda: R.save_snapshot(tmp, keyed.n_update, dict(loop=keyed.snapshot(), test=None), text,
                                                   args.n_env))
            save_s.append(dt)
        path = R.newest_snapshot(tmp)
        size = os.path.getsize(path)
        for _ in range(args.repeats):
            dt, _ = _timed(lambda: R.save_snapshot(tmp, keyed.n_update, dict(loop=keyed.snapshot(), test=None), text,
                                                   args.n_env))
            save_s.append(dt)
            _, fresh = _trainer(args.n_env)
            dt, _ = _timed(lambda: fresh.restore(R.load_snapshot(path)['run']['loop']))
            load_s.append(dt)
            assert torch.equal(fresh.engine.params, keyed.engine.params)
            del fresh
    print(json.dumps(dict(measure='snapshot', n_env=args.n_env, bytes=size,
                          write_s_median=statistics.median(save_s), write_s=save_s,
                          restore_s_median=statistics.median(load_s), restore_s=load_s)), flush=True)
    print(json.dumps(dict(measure='update', n_env=args.n_env, updates_per_round=args.updates,
                          without_ms=1e3 * statistics.median(per['without']),
                          with_ms=1e3 * statistics.median(per['with']),
                          without_rounds_ms=[1e3 * x for x in per['without']],
                          with_rounds_ms=[1e3 * x for x in per['with']])), flush=True)
    plain.graph = keyed.graph = None


if __name__ == '__main__':
    main_()
