"""NumPy restatement of nmarl_cacc_draw_par (per-env CACC scenario parameters) and the float64 oracle env of one row of
the table.

The draw, as include/nmarl.h documents it: Philox4x32-10 with key = seed, lane = env, stream tag 0x454E5650 and counter
= episode << 8 | k.  k = 0..6 draw the fields h_star, v_star, h_s, h_g, v_max, u_min, u_max as lo + u * (hi - lo);
k = 7 draws the scenario, slow-down iff u < slowdown_prob (no slowdown_prob: the config's scenario for every env).
The uniform is NumPy's 53-bit recipe on output words 0 and 1 (philox_ref.u01_from_bits).
"""
import numpy as np

from philox_ref import philox_u01
from oracle.cacc import OracleCACC

PAR_STREAM = 0x454E5650
FIELDS = ('h_star', 'v_star', 'h_s', 'h_g', 'v_max', 'u_min', 'u_max')
CATCHUP, SLOWDOWN = 0, 1


def draw_par(seed, episode, ranges, slowdown_prob, scenario):
    """episode: [B] resets each env has seen before the one it is about to start; ranges: {field: (lo, hi)};
    slowdown_prob None or p; scenario: the config's (0 catch-up, 1 slow-down) -> {field: float64 [B], 'scenario':
    int32 [B]} for every env (a masked call keeps the rows of the other envs)."""
    episode = np.asarray(episode, dtype=np.uint64)
    B = len(episode)
    lane = np.arange(B, dtype=np.uint64)
    u = lambda k: philox_u01(seed, (episode << np.uint64(8)) | np.uint64(k), lane, PAR_STREAM)
    out = {}
    for k, f in enumerate(FIELDS):
        lo, hi = (np.float64(x) for x in ranges[f])
        out[f] = lo + u(k) * (hi - lo)
    if slowdown_prob is None:
        out['scenario'] = np.full(B, scenario, dtype=np.int32)
    else:
        out['scenario'] = np.where(u(len(FIELDS)) < slowdown_prob, SLOWDOWN, CATCHUP).astype(np.int32)
    return out


def row(table, b):
    """Env b's parameters as a plain dict."""
    return {k: (int(v[b]) if k == 'scenario' else float(v[b])) for k, v in table.items()}


def oracle_env(env_config, par):
    """The float64 oracle env constructed with one env's parameter values: the reference CACCEnv reads these eight
    values from its config and nothing else from it differs."""
    o = OracleCACC(env_config)
    for f in FIELDS:
        setattr(o, f, par[f])
    o.name = 'slowdown' if par['scenario'] == SLOWDOWN else 'catchup'
    return o
