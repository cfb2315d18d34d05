"""Training one configuration on several processes (torchrun, one node): which envs and test seeds a rank owns, the
process group, and the gathers that let rank 0 write the records a one-process run of the same config writes.

Rank r of W owns the global envs [r * n_env / W, (r + 1) * n_env / W) of ENV_CONFIG.n_env and the contiguous part
[r * n / W, (r + 1) * n / W) of the n test seeds.  The kernels key every random draw by the global env index, so a
shard draws what the same envs of one process draw; the gradient is summed over the ranks (PolicyEngine.apply).
"""
import os

import torch

from . import _lib as L


def launch_world():
    """(world size, rank, local rank) that torchrun set for this process; (1, 0, 0) without torchrun."""
    return tuple(int(os.environ.get(k, d)) for k, d in (('WORLD_SIZE', 1), ('RANK', 0), ('LOCAL_RANK', 0)))


def world_rank():
    """(world size, rank) of the initialised process group; (1, 0) without one."""
    if torch.distributed.is_available() and torch.distributed.is_initialized():
        return torch.distributed.get_world_size(), torch.distributed.get_rank()
    return 1, 0


def env_shard(n_env, world, rank):
    """(env0, n_local): rank `rank` of `world` holds the global envs env0 .. env0 + n_local - 1 of the n_env envs.
    Raises ValueError for a split the batched loop cannot run: n_env = 1 (the one-env Trainer) on several ranks, or
    an n_env that the world size does not divide."""
    n_env, world, rank = int(n_env), int(world), int(rank)
    if world > 1 and n_env == 1:
        raise ValueError('ENV_CONFIG.n_env = 1 runs the one-env Trainer, which trains in one process only; '
                         'set n_env to a multiple of the %d processes' % world)
    if n_env < 1 or n_env % world:
        raise ValueError('ENV_CONFIG.n_env = %d (envs in total) must be a positive multiple of the %d processes'
                         % (n_env, world))
    per = n_env // world
    return rank * per, per


def seed_shard(seeds, world, rank):
    """The contiguous part of the test seeds that rank `rank` of `world` runs (may be empty)."""
    n = len(seeds)
    return list(seeds)[rank * n // world:(rank + 1) * n // world]


def init_from_env():
    """Under torchrun (WORLD_SIZE > 1): bind this process's GPU and initialise the process group from the environment.
    NCCL when every local rank has a GPU of its own; otherwise the ranks share GPUs and the group is gloo.  Returns the
    backend name, or None for one process."""
    world, _, local = launch_world()
    if world <= 1:
        return None
    L.require_cuda()
    local_world = int(os.environ.get('LOCAL_WORLD_SIZE', world))
    n_dev = torch.cuda.device_count()
    if n_dev >= local_world:
        torch.cuda.set_device(local)
        torch.distributed.init_process_group('nccl', device_id=torch.device('cuda', local))
        return 'nccl'
    torch.cuda.set_device(local % n_dev)
    torch.distributed.init_process_group('gloo')
    return 'gloo'


def gather_to_root(obj):
    """Every rank's picklable `obj` -> on rank 0 the list of them in rank order, None on the other ranks; [obj] with
    one process.  A host round trip: for records, not for the hot path."""
    world, rank = world_rank()
    if world == 1:
        return [obj]
    parts = [None] * world if rank == 0 else None
    torch.distributed.gather_object(obj, parts, dst=0)
    return parts


def concat_envs(parts, axes):
    """Per-env tensors of every rank ({name: tensor}, in rank order) -> the run's tensors in global env order, each
    concatenated along its env axis axes[name]."""
    return {k: torch.cat([p[k] for p in parts], dim=axes[k]) for k in parts[0]}


def take_envs(tensors, axes, env0, n):
    """The envs env0 .. env0 + n - 1 of per-env tensors in global env order ({name: tensor}, env axis axes[name])."""
    out = {}
    for k, t in tensors.items():
        if env0 < 0 or env0 + n > t.shape[axes[k]]:
            raise ValueError('%s holds %d envs, not the envs %d .. %d' % (k, t.shape[axes[k]], env0, env0 + n - 1))
        out[k] = t.narrow(axes[k], env0, n)
    return out


def check_replicas(tensors):
    """Raise RuntimeError on every rank unless all ranks hold bit-identical copies of the tensors {name: tensor}
    (the data-parallel replicas of the weights and optimizer state)."""
    world, _ = world_rank()
    if world == 1:
        return
    mine = {k: v.detach().cpu().numpy().tobytes() for k, v in tensors.items()}
    every = [None] * world
    torch.distributed.all_gather_object(every, mine)
    differ = sorted(k for k in mine if any(p[k] != every[0][k] for p in every))
    if differ:
        raise RuntimeError('data-parallel replicas differ across the %d ranks in: %s' % (world, ', '.join(differ)))


def shutdown():
    """Leave the process group: wait for this rank's device work, meet the other ranks, destroy the group."""
    if world_rank()[0] == 1:
        return
    torch.cuda.synchronize()
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


def _children():
    """{parent pid: [(pid, start time)]} of every process this user can see (/proc; Linux)."""
    out = {}
    for d in os.listdir('/proc'):
        if not d.isdigit():
            continue
        try:
            with open('/proc/%s/stat' % d) as f:
                fields = f.read().rsplit(')', 1)[1].split()
        except (OSError, IndexError):
            continue
        out.setdefault(int(fields[1]), []).append((int(d), fields[19]))      # ppid, starttime
    return out


def _descendants(pid):
    children, found, todo = _children(), [], [pid]
    while todo:
        for c in children.get(todo.pop(), []):
            found.append(c)
            todo.append(c[0])
    return found


def _start_time(pid):
    try:
        with open('/proc/%d/stat' % pid) as f:
            return f.read().rsplit(')', 1)[1].split()[19]
    except (OSError, IndexError):
        return None


def run_bounded(cmd, timeout, grace=60, **popen):
    """Run a command -- typically `python -m torch.distributed.run ... main.py ...` -- and return (exit code, output),
    or (None, output) when it did not finish within `timeout` seconds.  Nothing it started outlives the call: torchrun
    starts every worker in a session of its own, so on timeout the workers are listed first (before they can be
    re-parented), torchrun gets SIGTERM (it forwards the signal to its workers and escalates to SIGKILL) and `grace`
    seconds to stop them, and whatever is still alive then is killed.  The output goes through a file, so a worker
    that holds on to it cannot block the call."""
    import signal
    import subprocess
    import tempfile
    with tempfile.TemporaryFile('w+') as log:
        p = subprocess.Popen(cmd, stdout=log, stderr=subprocess.STDOUT, text=True, start_new_session=True, **popen)
        try:
            rc = p.wait(timeout=timeout)
        except subprocess.TimeoutExpired:
            rc = None
            procs = _descendants(p.pid)
            p.send_signal(signal.SIGTERM)
            try:
                p.wait(timeout=grace)
            except subprocess.TimeoutExpired:
                pass
            for pid, start in [(p.pid, _start_time(p.pid))] + procs:
                if start is not None and _start_time(pid) == start:          # the same process, not a reused pid
                    try:
                        os.kill(pid, signal.SIGKILL)
                    except ProcessLookupError:
                        pass
            p.wait()
        log.seek(0)
        return rc, log.read()
