"""What the 16-wide head costs: engine p-calls, v-calls and backward() + optimizer step at n_a = 4, 7 (8-wide head) and
8, 15 (16-wide head), NeurComm and DIAL on the 8-agent chain, B = 4096 envs, T = 60 steps, on both kernel families.

    python tools/bench_actions.py [--reps 10] [--warmup 3]

Prints one line per (agent, family, n_a): median milliseconds over --reps timed calls after --warmup untimed ones,
timed with CUDA events, plus the card name and power limit they were measured at."""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deeprl_network_b200 import _lib as L  # noqa: E402
from deeprl_network_b200.agents.engine import PolicyEngine  # noqa: E402
from deeprl_network_b200.layout import ModelLayout  # noqa: E402
from oracle.cacc import chain_masks  # noqa: E402

HP = dict(v_coef=0.5, e_coef=0.01, max_grad_norm=40.0, alpha=0.99, epsilon=1e-5, gamma=0.99, reward_norm=2000.0,
          reward_clip=-1.0)
N_ENV, T = 4096, 60


def _median_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def run(variant, n_a, tc, reps, warmup):
    mask = chain_masks(8)[0]
    lay = ModelLayout(variant, [5] * 8, n_a, mask)
    eng = PolicyEngine(lay, N_ENV, T, dict(HP), use_tc=tc)
    assert eng.use_tc == tc
    N, B = lay.N, N_ENV
    rs = np.random.RandomState(0)
    obs = torch.zeros(N, B, lay.obs_stride, device='cuda')
    obs[..., :5] = torch.as_tensor(rs.randn(N, B, 5).astype(np.float32), device='cuda')
    fp = torch.full((N, B, n_a), 1.0 / n_a, device='cuda')
    done = torch.zeros(B, device='cuda')
    pi = torch.zeros(N, B, n_a, device='cuda')
    act = torch.zeros(N, B, dtype=torch.int32, device='cuda')
    v = torch.zeros(N, B, device='cuda')
    # a recorded batch for backward(): random observations, actions, returns
    eng.T_cur = T
    eng.obs_buf[:T, :, :, :5].copy_(torch.as_tensor(rs.randn(T, N, B, 5).astype(np.float32)))
    eng.fp_buf[:T].fill_(1.0 / n_a)
    eng.act_buf.copy_(torch.as_tensor(rs.randint(0, n_a, size=(T, N, B)).astype(np.int32)))
    eng.done_buf[:T].copy_(torch.as_tensor((rs.rand(T, B) < 0.02).astype(np.float32)))
    eng.Rs.copy_(torch.as_tensor(rs.randn(T, N, B).astype(np.float32)))
    eng.Advs.copy_(torch.as_tensor(rs.randn(T, N, B).astype(np.float32)))

    def train():
        eng.backward()
        eng.apply(1e-4)
    p = _median_ms(lambda: eng.step_p(obs, fp, done, pi, act, L.SAMPLE_PHILOX), reps, warmup)
    vv = _median_ms(lambda: eng.step_v(obs, fp, done, act, v), reps, warmup)
    b = _median_ms(train, reps, warmup)
    eng.check_tc()
    return p, vv, b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    print('# %s; N = 8 (chain), B = %d, T = %d; median of %d after %d warm-up calls, ms' % (card, N_ENV, T, args.reps, args.warmup))
    print('%-10s %-6s %4s %3s %9s %9s %14s' % ('agent', 'family', 'n_a', 'HW', 'p-call', 'v-call', 'bwd+optim'))
    for variant in ('ma2c_nc', 'ma2c_dial'):
        for tc in (True, False):
            for n_a in (4, 7, 8, 15):
                p, v, b = run(variant, n_a, tc, args.reps, args.warmup)
                print('%-10s %-6s %4d %3d %9.3f %9.3f %14.3f' % (variant, 'tc' if tc else 'ffma', n_a, L.head_width(n_a), p, v, b),
                      flush=True)
                torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
