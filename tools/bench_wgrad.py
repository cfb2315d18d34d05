"""In-situ time of the weight-gradient GEMM (`tc_wgrad_kernel`) inside eagerly launched updates of the bench workload.

    python tools/bench_wgrad.py [--updates 20] [--n-env 4096] [--config config_ma2c_nc_catchup.ini] [--timeline]

Each update is launched eagerly (rollout, returns, backward, apply); CUDA events recorded on the backward stream
around the one `tc_wgrad_kernel` launch give its duration, as in `bench.py:kernel_rooflines`.  Prints median / min /
max over the updates with the card name and power limit.  --timeline additionally arms the kernel's clock64 stamps
(`nmarl_debug_set_prof`) for one more update and prints the per-k-block timeline of the first CTA of every job kind.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# stamp layout of tc_wgrad.cu (prof != NULL): one block of PROF_STRIDE int64 per job slot;
# [0] = start, [1] = number of k-blocks stamped, [2] = end, [3] = job kind | N << 8, then per k-block
# [B stage ready, A slot ready, MMAs retired]
PROF_STRIDE, PROF_HEAD = 1024, 4


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:                                 # the timing itself does not depend on it
        return 'unknown (%s)' % ex


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--updates', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--n-env', type=int, default=4096)
    ap.add_argument('--config', default='config_ma2c_nc_catchup.ini')
    ap.add_argument('--timeline', action='store_true', help='also print a per-k-block clock64 timeline per job kind')
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    from deeprl_network_b200 import _lib as L
    torch.cuda.set_device(0)
    _, env, model = bench.build(args.config, args.n_env, 0)
    e = model.engine
    assert e.use_tc, 'the weight-gradient GEMM runs on the tensor-core path only'
    from deeprl_network_b200.utils import VecTrainer
    vt = VecTrainer(env, model, graph=False, sample='philox')
    vt.start()
    e.overlap_v = False                                    # nothing else shares the SMs with the timed kernel
    mk = lambda: torch.cuda.Event(enable_timing=True)
    step_ev, wg_ev = [mk() for _ in range(2 * e.T)], [mk(), mk()]
    for ev in step_ev + wg_ev:
        ev.record()                                        # instantiates the cudaEvent_t handles

    def update(prof=None):
        e.rollout(env, sample=vt.sample)
        e.bwd_events = (step_ev, wg_ev)
        lib = L.lib()
        if prof is not None:
            lib.nmarl_debug_set_prof.argtypes = [C.c_void_p]
            lib.nmarl_debug_set_prof(prof.data_ptr())
        e.compute_returns(); e.backward()
        torch.cuda.synchronize()
        if prof is not None:
            lib.nmarl_debug_set_prof(None)
        e.bwd_events = None
        us = 1e3 * wg_ev[0].elapsed_time(wg_ev[1])
        e.apply(5e-4); e.roll_buffers(); e.normalize_cur()
        return us

    for _ in range(args.warmup):
        update()
    t = np.array([update() for _ in range(args.updates)])
    e.check_tc()                                           # a timed-out pipeline wait would void the numbers
    print('card: %s' % card())
    print('workload: %s, %d envs x %d agents, n_step %d' % (args.config, e.B, e.N, e.T))
    print('tc_wgrad_kernel in situ over %d eager updates: median %.1f us, min %.1f us, max %.1f us' %
          (len(t), np.median(t), t.min(), t.max()))
    if args.timeline:
        prof = torch.zeros(8 * PROF_STRIDE, dtype=torch.int64, device='cuda')
        update(prof)
        p = prof.cpu().numpy()
        for j in range(8):
            blk = p[j * PROF_STRIDE:(j + 1) * PROF_STRIDE]
            n = int(blk[1])
            if blk[0] == 0:
                continue
            t0 = blk[0]
            print('job slot %d (kind %d, N %d, first CTA of split 0, agent 0): %d k-blocks, %d cycles in all' %
                  (j, blk[3] & 0xFF, blk[3] >> 8, n, blk[2] - t0))
            st = blk[PROF_HEAD:PROF_HEAD + 3 * n].reshape(n, 3) - t0
            prev = np.concatenate([[0], st[:-1, 2]])
            for q in range(min(n, 4)):
                print('  q=%3d  B ready %8d  A ready %8d  retired %8d' % (q, st[q, 0], st[q, 1], st[q, 2]))
            if n > 8:
                s = slice(4, n)
                print('  k-blocks 4..%d, mean cycles: B wait %.0f, then A wait %.0f, MMAs + retire %.0f, '
                      'retire to retire %.0f' % (n - 1, np.mean(st[s, 0] - prev[s]), np.mean(st[s, 1] - st[s, 0]),
                                                 np.mean(st[s, 2] - st[s, 1]), np.mean(st[s, 2] - prev[s])))


if __name__ == '__main__':
    main()
