"""Agent-count scaling of the training step: NeurComm (ma2c_nc) catch-up at N = 8, 32, 64, 128 agents.

    python tools/bench_agents.py [--agents 8,32,64,128] [--agent-envs 32768] [--steps 10] [--warmup 2]

Every point keeps B * N = --agent-envs (B = 4096 envs at N = 8 ... 256 at N = 128), so each runs the same number of
agent rows per kernel and the same agent-env-steps per update; what changes is how the work is cut: more, smaller
per-agent groups, a larger model descriptor, a longer env chain.  The workload is bench.py's: whole updates
(rollout + returns + backward + clip / RMSProp) captured in a CUDA graph by VecTrainer, timed with CUDA events.
`kernels_per_update` counts the device kernels of one eager (uncaptured) update with torch.profiler.

Prints one JSON line per agent count plus a header line with the GPU name and its power limit.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    import torch
    info = {'gpu': torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info['power_limit'], info['max_sm_clock'] = [x.strip() for x in q.split(',')]
    except Exception as e:                       # noqa: BLE001 -- informational only
        info['power_limit'] = 'unknown (%s)' % e
    return info


def kernels_per_update(vt):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        vt.update()
        torch.cuda.synchronize()
    return sum(1 for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and 'Memcpy' not in ev.name
               and 'Memset' not in ev.name)


def run(n_agent, agent_envs, steps, warmup, config):
    import torch
    import main
    from deeprl_network_b200.utils import VecTrainer
    B = agent_envs // n_agent
    cfg = main.read_config(os.path.join(ROOT, 'config', config))
    cfg['ENV_CONFIG']['n_vehicle'] = str(n_agent)
    cfg['ENV_CONFIG']['n_env'] = str(B)
    env = main.init_env(cfg['ENV_CONFIG'])
    model = main.init_agent(env, cfg['MODEL_CONFIG'], 10 ** 9, cfg.getint('ENV_CONFIG', 'seed'))
    e = model.engine
    eager = VecTrainer(env, model, graph=False, sample='philox')
    eager.start()
    eager.update()
    kernels = kernels_per_update(eager)
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
    per_update = e.T * B * n_agent
    return {'agents': n_agent, 'envs': B, 'n_step': e.T, 'tensor_core_path': bool(e.use_tc),
            'agent_env_steps_per_s': steps * per_update / (ms * 1e-3), 'ms_per_update': ms / steps,
            'kernels_per_update': kernels}


def main_():
    ap = argparse.ArgumentParser()
    ap.add_argument('--agents', default='8,32,64,128')
    ap.add_argument('--agent-envs', type=int, default=32768)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--config', default='config_ma2c_nc_catchup.ini')
    args = ap.parse_args()
    print(json.dumps(dict(gpu_info(), workload='%s, B * N = %d' % (args.config, args.agent_envs))), flush=True)
    for n in [int(x) for x in args.agents.split(',')]:
        print(json.dumps(run(n, args.agent_envs, args.steps, args.warmup, args.config)), flush=True)


if __name__ == '__main__':
    main_()
