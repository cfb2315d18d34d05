"""Where one update goes: CUDA-event times of the phases of VecTrainer._one_update on the bench workload
(eager launches, so the numbers include launch gaps the captured graph does not have -- use them as a map,
not as the bench value).  Usage: python tools/phase_times.py [--n-env 4096] [--iters 5]"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from helpers import load_cfg  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='config_ma2c_nc_catchup.ini')
    ap.add_argument('--n-env', type=int, default=4096)
    ap.add_argument('--iters', type=int, default=5)
    args = ap.parse_args()
    import main as M
    from deeprl_network_b200 import _lib as L
    from deeprl_network_b200.envs.cacc_env import CACCEnv
    from deeprl_network_b200.utils import VecTrainer
    import ctypes as C
    cp = load_cfg(args.config, n_env=args.n_env)
    env = CACCEnv(cp['ENV_CONFIG'])
    np.random.seed(12)
    model = M.init_agent(env, cp['MODEL_CONFIG'], 10 ** 9, 12)
    vt = VecTrainer(env, model, graph=False)
    vt.start()
    e = model.engine
    for _ in range(2):
        vt.update()
    torch.cuda.synchronize()
    names = ['rollout', 'returns', 'heads', 'bptt', 'apply', 'episode']
    acc = {n: 0.0 for n in names}
    for _ in range(args.iters):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(names) + 1)]
        ev[0].record()
        e.rollout(env, sample=vt.sample)
        ev[1].record()
        e.compute_returns()
        ev[2].record()
        a = e._bwd_args(e.T_cur)
        assert getattr(e, 'saved_rollout', False), 'phase map assumes the fused-save rollout'
        ev[3].record()                      # 'heads' is part of the BPTT call (side stream)
        L.check(L.lib().nmarl_a2c_bptt(C.byref(e.model), C.byref(a), L.stream()), 'bptt')
        e.saved_rollout = False
        ev[4].record()
        e.apply(e.lr_dev)
        ev[5].record()
        done = e.done_buf[e.T_cur]
        e.roll_buffers(); e.reset_states(mask=done)
        env.reset_device(u01=None, mask=done, obs_out=e.obs_buf[0], fp_out=e.fp_buf[0], philox_seed=vt._seed)
        e.normalize_cur()
        ev[6].record()
        torch.cuda.synchronize()
        for k, n in enumerate(names):
            acc[n] += ev[k].elapsed_time(ev[k + 1])
    tot = sum(acc.values()) / args.iters
    print('phase times, eager launches, %d envs x %d agents x %d steps:' % (e.B, e.N, e.T))
    for n in names:
        print('  %-8s %7.3f ms  %5.1f%%' % (n, acc[n] / args.iters, 100 * acc[n] / args.iters / tot))
    print('  %-8s %7.3f ms' % ('total', tot))


if __name__ == '__main__':
    main()
