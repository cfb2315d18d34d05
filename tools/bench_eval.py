"""Cost of greedy evaluation episodes: per-seed Evaluator against the batched BatchedEvaluator.

    python tools/bench_eval.py [--config config_ma2c_nc_catchup.ini] [--n-env 4096] [--updates 10]

1. `main.py evaluate`'s core for the 50 default seeds: Evaluator.run (one env, one seed after the other) against
   BatchedEvaluator.run (all seeds in one pass), both writing the two CSV files to a temporary directory.  The
   batched call is timed cold (first call: builds the 50-env runner, eager launches), as `evaluate` runs it once.
   The files are compared byte for byte.
2. One TRAIN_CONFIG.greedy_test record against one update at the headline shape (4096 envs x 8 agents, NeurComm
   catch-up, CUDA-graph updates as bench.py runs them): log_test over the config's test seeds and over the 50
   default seeds, first call (eager) and later calls (replayed CUDA graph), each ending in its host sync.

Prints a header line with the GPU name and its power limit, then one JSON line per measurement.  Writes only to a
temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_agents import gpu_info  # noqa: E402


def _files(d):
    return {f: open(os.path.join(d, f), 'rb').read() for f in sorted(os.listdir(d))}


def evaluate_core(config):
    import torch
    import main
    from deeprl_network_b200 import utils as U
    seeds = [int(s) for s in main.DEFAULT_EVAL_SEEDS.split(',')]
    cfg = main.read_config(os.path.join(ROOT, 'config', config))
    cfg['ENV_CONFIG']['n_env'] = '1'
    env = main.init_env(cfg['ENV_CONFIG'])
    model = main.init_agent(env, cfg['MODEL_CONFIG'], 0, 0)
    with tempfile.TemporaryDirectory() as one, tempfile.TemporaryDirectory() as many:
        env.init_test_seeds(seeds)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        U.Evaluator(env, model, one + '/').run()
        t1 = time.perf_counter()
        U.BatchedEvaluator(cfg['ENV_CONFIG'], model, many + '/').run(seeds)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        same = _files(one) == _files(many)
    return {'measure': 'evaluate_core', 'config': config, 'seeds': len(seeds), 'per_seed_s': t1 - t0,
            'batched_s': t2 - t1, 'speedup': (t1 - t0) / (t2 - t1), 'files_identical': same}


def greedy_test_cost(config, n_env, updates):
    import torch
    import main
    from deeprl_network_b200 import utils as U
    cfg = main.read_config(os.path.join(ROOT, 'config', config))
    cfg['ENV_CONFIG']['n_env'] = str(n_env)
    env = main.init_env(cfg['ENV_CONFIG'])
    model = main.init_agent(env, cfg['MODEL_CONFIG'], 10 ** 9, cfg.getint('ENV_CONFIG', 'seed'))
    vt = U.VecTrainer(env, model, graph=True)
    vt.start()
    for _ in range(3):
        vt.update()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(updates):
        vt.update()
    torch.cuda.synchronize()
    upd = (time.perf_counter() - t0) / updates
    out = []
    for name, seeds in (('config_test_seeds', env.test_seeds),
                        ('default_eval_seeds', [int(s) for s in main.DEFAULT_EVAL_SEEDS.split(',')])):
        tester = U.BatchedEvaluator(cfg['ENV_CONFIG'], model)
        times = []
        for k in range(5):                      # call 0: eager; call 1 captures the graph; 2.. replay it
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tester.log_test(k, seeds)
            times.append(time.perf_counter() - t0)
        replay = sum(times[2:]) / len(times[2:])
        out.append({'measure': 'greedy_test_record', 'config': config, 'envs': n_env, 'agents': env.n_agent,
                    'test_seeds': name, 'n_seeds': len(seeds), 'ms_per_update': upd * 1e3,
                    'ms_first_record_eager': times[0] * 1e3, 'ms_record_graph': replay * 1e3,
                    'record_over_update': replay / upd})
    return out


def main_():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='config_ma2c_nc_catchup.ini')
    ap.add_argument('--n-env', type=int, default=4096)
    ap.add_argument('--updates', type=int, default=10)
    args = ap.parse_args()
    print(json.dumps(dict(gpu_info(), workload='%s, %d envs' % (args.config, args.n_env))), flush=True)
    print(json.dumps(evaluate_core(args.config)), flush=True)
    for r in greedy_test_cost(args.config, args.n_env, args.updates):
        print(json.dumps(r), flush=True)


if __name__ == '__main__':
    main_()
