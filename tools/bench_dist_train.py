"""Wall time per update of `main.py train` in one process and in several processes (torchrun).

    python tools/bench_dist_train.py [--config config/config_ma2c_nc_catchup.ini] [--envs 4096] [--updates 30]
                                     [--out DIR]

Runs the command line a user runs and reads the timestamps of rank 0's per-update log lines (with n_step x n_env
larger than log_interval every update logs one record, which includes its host sync and the gather to rank 0): the
mean time between consecutive records after the first three updates is the wall time per update.  Measured:
  * one process, `--envs` envs;
  * two gloo ranks sharing the first GPU, `--envs` envs in total (what the eager fall-back costs);
  * with at least 2 / 4 GPUs: 2 and 4 NCCL ranks with `--envs` envs PER GPU (weak scaling; 1 rank is the first line).
Prints one JSON line per run, each with the GPU's name and power limit read in the same call.
"""
import argparse
import configparser
import datetime
import glob
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deeprl_network_b200.dist import run_bounded  # noqa: E402
STAMP = re.compile(r'^(\d{4}-\d\d-\d\d \d\d:\d\d:\d\d,\d{3}) .*update (\d+), env steps \d+, mean step reward')


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    return [line.strip() for line in q.stdout.strip().split('\n')] if q.returncode == 0 else ['unknown']


def run(tmp, cfg_path, envs, updates, procs, one_gpu):
    cp = configparser.ConfigParser()
    cp.read(cfg_path)
    T = cp.getint('MODEL_CONFIG', 'batch_size')
    cp['ENV_CONFIG']['n_env'] = str(envs)
    cp['TRAIN_CONFIG']['total_step'] = str(updates * T * envs)
    cp['TRAIN_CONFIG']['log_interval'] = '1'
    tag = '%s%d_%d' % ('gloo' if one_gpu and procs > 1 else 'p', procs, envs)
    ini, base = os.path.join(tmp, tag + '.ini'), os.path.join(tmp, tag)
    with open(ini, 'w') as f:
        cp.write(f)
    env = dict(os.environ)
    if one_gpu:
        env['CUDA_VISIBLE_DEVICES'] = env.get('CUDA_VISIBLE_DEVICES', '0').split(',')[0] or '0'
    main = os.path.join(ROOT, 'main.py')
    cmd = [sys.executable, main] if procs == 1 else \
        [sys.executable, '-m', 'torch.distributed.run', '--standalone', '--nproc-per-node', str(procs), main]
    # on timeout torchrun and every worker it started are stopped: nothing is left on the GPUs
    rc, out = run_bounded(cmd + ['--base-dir', base, 'train', '--config-dir', ini], 1800, env=env)
    if rc != 0:
        raise RuntimeError('%s %s:\n%s' % (tag, 'timed out' if rc is None else 'failed (exit %d)' % rc, out[-6000:]))
    times = []
    for f in glob.glob(os.path.join(base, 'log', '*.log')):
        for line in open(f):
            m = STAMP.match(line)
            if m:
                times.append((int(m.group(2)), datetime.datetime.strptime(m.group(1), '%Y-%m-%d %H:%M:%S,%f')))
    times.sort()
    times = [t for u, t in times if u > 3]
    ms = (times[-1] - times[0]).total_seconds() * 1e3 / (len(times) - 1)
    return {'run': tag, 'processes': procs, 'backend': 'gloo' if one_gpu and procs > 1 else
            ('nccl' if procs > 1 else None), 'envs_total': envs, 'updates_timed': len(times) - 1,
            'ms_per_update': round(ms, 2), 'gpus': gpu_info()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    ap.add_argument('--config', default=os.path.join(ROOT, 'config', 'config_ma2c_nc_catchup.ini'))
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--updates', type=int, default=30)
    ap.add_argument('--out', default=None, help='also append the JSON lines to DIR/bench_dist_train.jsonl')
    args = ap.parse_args()
    import torch
    n_gpu = torch.cuda.device_count()
    plan = [(args.envs, 1, True), (args.envs, 2, True)]
    plan += [(args.envs * k, k, False) for k in (2, 4) if n_gpu >= k]
    with tempfile.TemporaryDirectory() as tmp:
        for envs, procs, one_gpu in plan:
            r = run(tmp, args.config, envs, args.updates, procs, one_gpu)
            line = json.dumps(r)
            print(line, flush=True)
            if args.out:
                os.makedirs(args.out, exist_ok=True)
                with open(os.path.join(args.out, 'bench_dist_train.jsonl'), 'a') as f:
                    f.write(line + '\n')
    if n_gpu < 2:
        print(json.dumps({'nccl': 'not measured: %d GPU visible' % n_gpu}))


if __name__ == '__main__':
    main()
