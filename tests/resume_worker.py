"""One process of a batched training run that takes or restores a snapshot; tests/test_gpu_resume.py runs it under
torchrun (ranks sharing one GPU over gloo) and imports its helpers for the one-process side.

    python resume_worker.py INI OUT BEFORE AFTER [SNAPSHOT]

Without SNAPSHOT: BEFORE updates, then VecTrainer.snapshot -> OUT/snap.pt (rank 0) and this rank's own per-env state
-> OUT/local-<rank>.pt.  With SNAPSHOT: restore it and write this rank's restored per-env state to
OUT/restored-<rank>.pt.  Then AFTER more updates, each with a train_reward record; rank 0 writes the parameters, the
RMSProp state and the records to OUT/end.pt, after checking that every rank holds the same parameters.
"""
import configparser
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import main  # noqa: E402
from deeprl_network_b200 import dist as D  # noqa: E402
from deeprl_network_b200 import utils as U  # noqa: E402


def build(ini):
    """The env, model and started VecTrainer of this process (one shard under torchrun)."""
    cp = configparser.ConfigParser()
    cp.read(ini)
    world, rank, _ = D.launch_world()
    shard = backend = None
    if world > 1:
        shard = D.env_shard(cp.getint('ENV_CONFIG', 'n_env'), world, rank)
        backend = D.init_from_env()
    env = main.init_env(cp['ENV_CONFIG'], shard=shard)
    kw = {} if shard is None else dict(env0=env.env0, n_env_total=env.n_env_total)
    model = main.init_agent(env, cp['MODEL_CONFIG'], int(cp.getfloat('TRAIN_CONFIG', 'total_step')),
                            cp.getint('ENV_CONFIG', 'seed'), **kw)
    loop = U.VecTrainer(env, model, graph=backend != 'gloo')
    loop.start()
    return loop


def local_state(loop):
    """This process's per-env tensors in the snapshot layout, {'engine.<name>' / 'env.<name>': tensor}, and their env
    axes."""
    state, axes = {}, {}
    for tag, snap in (('engine.', loop.engine.snapshot()), ('env.', loop.env.snapshot())):
        state.update({tag + k: v for k, v in snap['envs'].items()})
        axes.update({tag + k: a for k, a in snap['env_axis'].items()})
    return state, axes


def snapshot_state(snap):
    """The per-env tensors of a VecTrainer snapshot, named as local_state names them."""
    state = {'engine.' + k: v for k, v in snap['engine']['envs'].items()}
    state.update({'env.' + k: v for k, v in snap['env']['envs'].items()})
    return state


def run(loop, n):
    for _ in range(n):
        loop.update()
        loop.log_rewards(loop.n_update)


def main_(ini, out, before, after, snapshot=None):
    loop = build(ini)
    _, rank = D.world_rank()
    if snapshot is None:
        run(loop, before)
        snap = loop.snapshot()
        if snap is not None:
            torch.save(snap, os.path.join(out, 'snap.pt'))
        torch.save(local_state(loop)[0], os.path.join(out, 'local-%d.pt' % rank))
    else:
        loop.restore(torch.load(snapshot, map_location='cpu', weights_only=True))
        torch.save(local_state(loop)[0], os.path.join(out, 'restored-%d.pt' % rank))
    run(loop, after)
    e = loop.engine
    D.check_replicas({'params': e.params, 'rmsprop ms': e.ms})
    if rank == 0:
        torch.save(dict(params=e.params.cpu(), ms=e.ms.cpu(), data=U.plain_records(loop.data)),
                   os.path.join(out, 'end.pt'))
    loop.graph = None
    D.shutdown()


if __name__ == '__main__':
    a = sys.argv[1:]
    main_(a[0], a[1], int(a[2]), int(a[3]), a[4] if len(a) > 4 else None)
