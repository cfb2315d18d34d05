"""The files of a resumable training run: periodic snapshots next to the checkpoints under <base>/model/.

    checkpoint-<step>.pt   parameters and RMSProp state (IA2C.save; what `load` and `main.py evaluate` read)
    resume-<step>.pt       the run state VecTrainer.snapshot collects, the configuration text and the env count

Every file is written under a temporary name that starts with '.' in the same directory and then renamed over its
final name, so a process killed during a write leaves no file that either pattern picks up.  The newest KEEP of each
kind are kept, like the reference's tf.train.Saver(max_to_keep=5).
"""
import configparser
import os
import re

import torch

KEEP = 5
FORMAT = 1
CHECKPOINT_RE = re.compile(r'^checkpoint-(\d+)\.pt$')
RESUME_RE = re.compile(r'^resume-(\d+)\.pt$')
# the one key a resumed run may change: a larger total_step trains longer
FREE_KEYS = (('TRAIN_CONFIG', 'total_step'),)


def atomic_save(obj, path):
    """torch.save to a temporary file in the same directory, flushed to disk, then renamed over `path`."""
    d, name = os.path.split(path)
    tmp = os.path.join(d, '.%s.%d.tmp' % (name, os.getpid()))
    try:
        with open(tmp, 'wb') as f:
            torch.save(obj, f)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)


def _steps(model_dir, pattern):
    """{step: file name} of the files under model_dir whose whole name matches pattern."""
    if not os.path.isdir(model_dir):
        return {}
    return {int(m.group(1)): f for f in os.listdir(model_dir) for m in [pattern.match(f)] if m}


def newest_snapshot(model_dir):
    """Path of the resume-<step>.pt with the largest step under model_dir, or None."""
    found = _steps(model_dir, RESUME_RE)
    return os.path.join(model_dir, found[max(found)]) if found else None


def prune(model_dir, keep=KEEP):
    """Remove all but the newest `keep` checkpoint-<step>.pt and the newest `keep` resume-<step>.pt."""
    for pattern in (CHECKPOINT_RE, RESUME_RE):
        found = _steps(model_dir, pattern)
        for step in sorted(found)[:-keep]:
            os.remove(os.path.join(model_dir, found[step]))


def save_snapshot(model_dir, step, snap, config_text, n_env):
    """Write <model_dir>/resume-<step>.pt: the run state `snap`, the configuration text and the run's env count."""
    atomic_save(dict(format=FORMAT, step=int(step), config=config_text, n_env=int(n_env), run=snap),
                os.path.join(model_dir, 'resume-%d.pt' % int(step)))


def load_snapshot(path):
    snap = torch.load(path, map_location='cpu', weights_only=True)
    if snap.get('format') != FORMAT:
        raise ValueError('%s is not a snapshot this version writes (format %r)' % (path, snap.get('format')))
    return snap


def _parse(text):
    cp = configparser.ConfigParser(interpolation=None)
    cp.read_string(text)
    return cp


def config_difference(saved_text, text):
    """The first key (as 'SECTION.key', with both values) in which two configuration texts differ, apart from
    FREE_KEYS; None when they agree."""
    a, b = _parse(saved_text), _parse(text)
    for sec in sorted(set(a.sections()) | set(b.sections())):
        ka = dict(a[sec]) if a.has_section(sec) else {}
        kb = dict(b[sec]) if b.has_section(sec) else {}
        for key in sorted(set(ka) | set(kb)):
            if (sec, key) not in FREE_KEYS and ka.get(key) != kb.get(key):
                return '%s.%s' % (sec, key), ka.get(key), kb.get(key)
    return None


def check_resumable(snap, config_text, n_env):
    """Raise ValueError unless a run of this configuration text with n_env envs in total may continue the snapshot."""
    if int(snap['n_env']) != int(n_env):
        raise ValueError('--resume: the snapshot holds %d envs in total and ENV_CONFIG.n_env is %d; a run continues '
                         'with the env count it started with' % (int(snap['n_env']), int(n_env)))
    diff = config_difference(snap['config'], config_text)
    if diff is not None:
        raise ValueError('--resume: %s is %r in the snapshot and %r in the configuration; only %s may change' % (
            diff + (', '.join('%s.%s' % k for k in FREE_KEYS),)))
