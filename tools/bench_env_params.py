"""Cost of per-env CACC scenario parameters (ENV_CONFIG <key>_range / slowdown_prob).

    python tools/bench_env_params.py [--config config_ma2c_nc_catchup.ini] [--n-env 4096] [--launches 2000]
                                     [--updates 10] [--rounds 4]

Three variants of the config: `nominal` (no key: nmarl_cacc_step / nmarl_cacc_reset), `point` (every key given as
the point range of its nominal value and slowdown_prob 0 or 1 for the config's scenario: the *_pe kernels, every env
exactly the nominal env) and `open` (every range open, slowdown_prob 0.5).  `point` - `nominal` is the cost of the
per-env table; `open` - `point` is what heterogeneous envs cost on top (warps whose lanes follow different branches).

1. The env step alone on n_env x 8 agents, random actions.  Each launch is timed with its own pair of CUDA events;
   the median over `launches` launches per variant, the variants alternating in blocks of 100 launches.  The envs
   are reset (untimed) every 600 steps.  Also the reset of every env (draw + reset for the *_pe variants).
2. One NeurComm update (rollout + BPTT + RMSProp, replayed CUDA graph as bench.py runs it) per variant: `rounds`
   alternating rounds of `updates` updates each, median of the per-round means.

Prints a header line with the GPU name and its power limit, then one JSON line per measurement.  Writes nothing.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_agents import gpu_info  # noqa: E402

OPEN = dict(headway_target_range='15, 25', speed_target_range='12, 18', headway_st_range='3, 7',
            headway_go_range='30, 40', speed_max_range='25, 35', accel_min_range='-3, -2',
            accel_max_range='2, 3', slowdown_prob='0.5')


VARIANTS = ('nominal', 'point', 'open')


def _cfg(config, n_env, variant):
    import main
    cfg = main.read_config(os.path.join(ROOT, 'config', config))
    sec = cfg['ENV_CONFIG']
    sec['n_env'] = str(n_env)
    if variant == 'point':
        for k in OPEN:
            if k.endswith('_range'):
                sec[k] = '%s, %s' % (sec[k[:-6]], sec[k[:-6]])
        sec['slowdown_prob'] = '1' if 'slowdown' in sec['scenario'] else '0'
    elif variant == 'open':
        sec.update(OPEN)
    return cfg


def env_step_cost(config, n_env, launches):
    import torch
    import main
    envs = {k: main.init_env(_cfg(config, n_env, k)['ENV_CONFIG']) for k in VARIANTS}
    N = envs['nominal'].n_agent
    g = torch.Generator(device='cuda').manual_seed(0)
    acts = [torch.randint(0, 4, (N, n_env), dtype=torch.int32, device='cuda', generator=g) for _ in range(64)]
    steps = {k: 0 for k in envs}
    times = {k: [] for k in envs}
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(100)]
    for e in envs.values():
        e.reset_device(u01=None, philox_seed=12)
    for _ in range(2):                                       # warm-up block of each
        for k, e in envs.items():
            for i in range(100):
                e.step_device(acts[i % 64])
    while min(len(v) for v in times.values()) < launches:
        for k, e in envs.items():
            for i in range(100):
                if steps[k] % 600 == 0:
                    e.reset_device(u01=None, philox_seed=12 + steps[k])
                ev[i][0].record()
                e.step_device(acts[steps[k] % 64])
                ev[i][1].record()
                steps[k] += 1
            torch.cuda.synchronize()
            times[k].extend(a.elapsed_time(b) * 1e3 for a, b in ev)
    rst = {}
    for k, e in envs.items():
        t = []
        for _ in range(200):
            ev[0][0].record()
            e.reset_device(u01=None, philox_seed=5)
            ev[0][1].record()
            torch.cuda.synchronize()
            t.append(ev[0][0].elapsed_time(ev[0][1]) * 1e3)
        rst[k] = statistics.median(t)
    med = {k: statistics.median(v) for k, v in times.items()}
    return [dict({'measure': 'env_step', 'envs': n_env, 'agents': N, 'launches': len(times['nominal'])},
                 **{'us_' + k: med[k] for k in VARIANTS}),
            dict({'measure': 'env_reset_all', 'envs': n_env, 'agents': N}, **{'us_' + k: rst[k] for k in VARIANTS})]


def update_cost(config, n_env, updates, rounds):
    import torch
    import main
    from deeprl_network_b200 import utils as U
    loops = {}
    for k in VARIANTS:
        cfg = _cfg(config, n_env, k)
        env = main.init_env(cfg['ENV_CONFIG'])
        model = main.init_agent(env, cfg['MODEL_CONFIG'], 10 ** 9, cfg.getint('ENV_CONFIG', 'seed'))
        vt = U.VecTrainer(env, model, graph=True)
        vt.start()
        for _ in range(3):
            vt.update()
        loops[k] = vt
    torch.cuda.synchronize()
    per = {k: [] for k in loops}
    for _ in range(rounds):
        for k, vt in loops.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(updates):
                vt.update()
            torch.cuda.synchronize()
            per[k].append((time.perf_counter() - t0) / updates * 1e3)
    med = {k: statistics.median(v) for k, v in per.items()}
    return dict({'measure': 'update', 'config': config, 'envs': n_env, 'updates_per_round': updates, 'rounds': rounds},
                **{'ms_' + k: med[k] for k in VARIANTS},
                **{'share_' + k: med[k] / med['nominal'] - 1 for k in VARIANTS[1:]},
                **{'ms_rounds_' + k: per[k] for k in VARIANTS})


def main_():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='config_ma2c_nc_catchup.ini')
    ap.add_argument('--n-env', type=int, default=4096)
    ap.add_argument('--launches', type=int, default=2000)
    ap.add_argument('--updates', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=4)
    args = ap.parse_args()
    print(json.dumps(dict(gpu_info(), workload='%s, %d envs' % (args.config, args.n_env))), flush=True)
    for r in env_step_cost(args.config, args.n_env, args.launches):
        print(json.dumps(r), flush=True)
    print(json.dumps(update_cost(args.config, args.n_env, args.updates, args.rounds)), flush=True)


if __name__ == '__main__':
    main_()
