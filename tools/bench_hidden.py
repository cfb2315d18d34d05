"""Training throughput against the LSTM width: NeurComm (ma2c_nc) catch-up, 4096 envs x 8 agents, n_step = 60.

    python tools/bench_hidden.py [--widths 16,32,64,64-ffma] [--n-env 4096] [--steps 10] [--warmup 3]

Widths 16 and 32 run the FP32-FFMA kernels (the tensor-core kernels are built for num_lstm = 64 only).  64 runs the
tensor-core path, as bench.py does; "64-ffma" runs width 64 with NMARL_NO_TC=1, the FFMA kernels, so that the narrow
widths have a like-for-like comparison.  The workload is bench.py's: whole updates (rollout + returns + backward +
clip / RMSProp) captured in a CUDA graph by VecTrainer, timed with CUDA events after the warm-up updates.

Prints a header line with the GPU name and its power limit, then one JSON line per width.  Writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_agents import gpu_info  # noqa: E402


def run(width, n_env, steps, warmup, config):
    import torch
    import main
    from deeprl_network_b200.utils import VecTrainer
    n_h = int(width.split('-')[0])
    cfg = main.read_config(os.path.join(ROOT, 'config', config))
    cfg['ENV_CONFIG']['n_env'] = str(n_env)
    cfg['MODEL_CONFIG']['num_lstm'] = str(n_h)
    cfg['MODEL_CONFIG']['num_fc'] = str(n_h)
    old = os.environ.get('NMARL_NO_TC')
    os.environ['NMARL_NO_TC'] = '1' if width.endswith('-ffma') else '0'
    try:
        env = main.init_env(cfg['ENV_CONFIG'])
        model = main.init_agent(env, cfg['MODEL_CONFIG'], 10 ** 9, cfg.getint('ENV_CONFIG', 'seed'))
    finally:
        if old is None:
            del os.environ['NMARL_NO_TC']
        else:
            os.environ['NMARL_NO_TC'] = old
    e = model.engine
    vt = VecTrainer(env, model, graph=True, sample='philox')
    vt.start()
    for _ in range(max(1, warmup)):
        vt.update()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(steps):
        vt.update()
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1)
    assert torch.isfinite(e.params).all()
    return {'width': width, 'num_lstm': n_h, 'envs': n_env, 'agents': e.N, 'n_step': e.T,
            'tensor_core_path': bool(e.use_tc), 'agent_env_steps_per_s': steps * e.T * n_env * e.N / (ms * 1e-3),
            'ms_per_update': ms / steps}


def main_():
    ap = argparse.ArgumentParser()
    ap.add_argument('--widths', default='16,32,64,64-ffma')
    ap.add_argument('--n-env', type=int, default=4096)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--config', default='config_ma2c_nc_catchup.ini')
    args = ap.parse_args()
    print(json.dumps(dict(gpu_info(), workload='%s, %d envs' % (args.config, args.n_env))), flush=True)
    for w in args.widths.split(','):
        print(json.dumps(run(w, args.n_env, args.steps, args.warmup, args.config)), flush=True)


if __name__ == '__main__':
    main_()
