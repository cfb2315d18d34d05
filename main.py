"""Command line of the H100-native CACC / networked-A2C hot path.

The reference's command line is kept verbatim (main.py:21-40 there) so existing scripts keep working:

    python main.py --base-dir D train    --config-dir F.ini
    python main.py --base-dir D evaluate [--evaluation-seeds s1,s2,...] [--demo]

and so is the .ini surface (MODEL_CONFIG / TRAIN_CONFIG / ENV_CONFIG).  Optional new keys: ENV_CONFIG.n_env
(parallel episodes in total) and TRAIN_CONFIG.greedy_test (default false).  n_env = 1 runs the reference's
one-episode-at-a-time Trainer; n_env > 1 the device-resident VecTrainer, which with greedy_test also logs the greedy
test reward over ENV_CONFIG.test_seeds to data/test_reward.csv.  With n_env > 1, ENV_CONFIG.<key>_range / slowdown_prob
give every env its own scenario parameters, redrawn at each of its resets (data/env_par.csv records what was drawn);
evaluation keeps the nominal values.  evaluate runs all seeds at once on the device and
writes the files the reference's one-seed-at-a-time Evaluator writes.  Agents: ia2c, ia2c_fp, ma2c_cu, ma2c_nc, ma2c_ic3, ma2c_dial on the CACC scenarios;
ATSC/SUMO environments are out of scope (SURVEY row 10).

train also runs on all the GPUs of a node under torchrun, e.g. `torchrun --standalone --nproc-per-node 8 main.py
--base-dir D train --config-dir F.ini`: rank r of W trains the envs [r n_env / W, (r + 1) n_env / W) of ENV_CONFIG.n_env
and the gradient is summed over the ranks, which gives the training run of one process with the same .ini up to the
order of floating-point sums.  Rank 0 alone writes the log, the files under data/ and the checkpoint.  NCCL when every
rank has a GPU of its own, else gloo (ranks sharing a GPU; no CUDA graphs).  Refused with a ValueError: n_env not
divisible by the process count, n_env = 1, and evaluate under torchrun (INTEGRATION §4).

With n_env > 1 a run can survive its process.  TRAIN_CONFIG.checkpoint_interval (environment steps) makes rank 0 write
model/checkpoint-<step>.pt and the snapshot model/resume-<step>.pt at the first update boundary after each multiple
(the newest 5 of each are kept), and

    python main.py --base-dir D train --config-dir F.ini --resume

continues from the newest D/model/resume-*.pt, also under torchrun with another process count.  F.ini must equal the
snapshot's configuration except for a raised TRAIN_CONFIG.total_step; with lr_decay = linear the schedule's horizon is
the new total_step from the resume point on, so the rate jumps there to lr_init (1 - n / new total_step) and ramps down
to lr_min at the new end.  Refused with a ValueError on every rank: no snapshot, n_env = 1, an
n_env other than the snapshot's, and any other configuration difference (INTEGRATION §4, DESIGN §5.1).
"""
import argparse
import configparser
import logging
import os

from deeprl_network_b200.agents import models as agent_models
from deeprl_network_b200.envs.cacc_env import CACCEnv, nominal_config
from deeprl_network_b200 import dist as D
from deeprl_network_b200 import resume as R
from deeprl_network_b200 import utils as U

AGENTS = {'ia2c': agent_models.IA2C, 'ia2c_fp': agent_models.IA2C_FP, 'ma2c_cu': agent_models.IA2C_CU,
          'ma2c_nc': agent_models.MA2C_NC, 'ma2c_ic3': agent_models.MA2C_IC3, 'ma2c_dial': agent_models.MA2C_DIAL}
DEFAULT_EVAL_SEEDS = ','.join(str(s) for s in range(2000, 2500, 10))


def parse_args(argv=None):
    top = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    top.add_argument('--base-dir', type=str, default='./runs/ma2c_nc_catchup', help='experiment base dir')
    modes = top.add_subparsers(dest='option', help='train or evaluate')
    tr = modes.add_parser('train', help='train the agent named in the config under the base dir')
    tr.add_argument('--config-dir', type=str, default='./config/config_ma2c_nc_catchup.ini', help='experiment config path')
    tr.add_argument('--resume', action='store_true',
                    help='continue from the newest snapshot <base-dir>/model/resume-<step>.pt (n_env > 1)')
    ev = modes.add_parser('evaluate', help='evaluate the agent stored under the base dir')
    ev.add_argument('--evaluation-seeds', type=str, default=DEFAULT_EVAL_SEEDS, help='random seeds for evaluation, split by ,')
    ev.add_argument('--demo', action='store_true', help='accepted for compatibility (SUMO gui in the reference); no files are written')
    args = top.parse_args(argv)
    if args.option is None:
        top.print_help()
        raise SystemExit(1)
    return args


def read_config(path):
    cfg = configparser.ConfigParser()
    if not cfg.read(path):
        raise FileNotFoundError(path)
    return cfg


def init_env(config, port=0, shard=None):
    """ENV_CONFIG section -> environment (only the CACC family exists here).  shard: (env0, n_env) of this process
    in a run over several processes (ENV_CONFIG.n_env is then the run's total)."""
    if config.get('scenario').startswith('atsc'):
        raise NotImplementedError('ATSC/SUMO environments are outside the accelerated hot path')
    if shard is None:
        return CACCEnv(config)
    return CACCEnv(config, n_env=shard[1], env0=shard[0], n_env_total=config.getint('n_env'))


def init_agent(env, config, total_step, seed, **kw):
    """MODEL_CONFIG section -> agent object of the class ENV_CONFIG.agent names (None if unknown)."""
    if env.agent not in AGENTS:
        logging.error('agent %r is not on the accelerated hot path' % env.agent)
        return None
    # device-resident rollouts (n_env > 1 in the run, kw n_env_total for one shard of it) gather neighbour
    # observations in the kernel
    if env.agent == 'ia2c' and kw.get('n_env_total', env.n_env) > 1:
        kw.setdefault('obs_mode', 'gather')
    return AGENTS[env.agent](env.n_s_ls, env.n_a_ls, env.neighbor_mask, env.distance_mask, env.coop_gamma,
                             total_step, config, seed=seed, n_env=env.n_env, **kw)


def _train_batched(env, model, total_step, log_interval, writer=None, output_path=None, tester=None, graph=True,
                   resume=None, checkpoint_interval=0, checkpoint=None):
    """n_env > 1: whole updates on the device until total_step environment steps (summed over all envs of all
    processes) are done.
    Every `log_interval` environment steps one record goes to data/train_reward.csv (and the TB scalar
    `train_reward`): mean / std of the per-step global TRAINING reward of the last batch.  With a `tester`
    (BatchedEvaluator, TRAIN_CONFIG.greedy_test) each record also runs one greedy episode per ENV_CONFIG test seed
    with the current weights and adds a record to data/test_reward.csv (and the TB scalar `test_reward`).  In a run over
    several processes every rank calls it; the records are taken on rank 0 (the others pass output_path None).
    resume: a snapshot's run state, put in place before the first update.  With a checkpoint_interval (environment
    steps), checkpoint(run state or None, env steps) is called at the first update boundary after each multiple."""
    loop = U.VecTrainer(env, model, graph=graph)
    loop.start()
    if resume is not None:
        loop.restore(resume['loop'])
        if tester is not None:
            tester.restore(resume['test'])
    per_update = model.n_step * env.n_env_total
    done_steps = loop.n_update * per_update
    every = max(1, int(log_interval) // per_update)

    def log():
        r = loop.log_rewards(done_steps, writer)
        if r is not None:
            logging.info('update %d, env steps %d, mean step reward %.2f' % (loop.n_update, done_steps, r))
        if tester is not None:
            r = tester.log_test(done_steps, env.test_seeds, writer)
            if r is not None:
                logging.info('update %d, env steps %d, greedy test reward %.2f' % (loop.n_update, done_steps, r))
    while done_steps < total_step:
        loop.update()
        done_steps += per_update
        on_cadence = loop.n_update % every == 0
        if on_cadence:
            log()
        if checkpoint_interval and done_steps // checkpoint_interval > (done_steps - per_update) // checkpoint_interval:
            run = loop.snapshot()                  # every rank takes part; rank 0 gets the run state
            if run is not None:
                checkpoint(dict(loop=run, test=None if tester is None else tester.snapshot()), done_steps)
        if not on_cadence and done_steps >= total_step:
            # the last update's record, off the cadence: taken after the snapshot, so that a run resumed from it (and
            # trained longer) writes the records of the uninterrupted run
            log()
    if output_path is not None:
        loop.write_csv(output_path)
        if tester is not None:
            tester.write_csv(output_path)
    loop.graph = None          # a captured graph may hold NCCL kernels: release it before the process group goes
    return done_steps


def _resume_state(args, config_text, n_env):
    """--resume: the newest snapshot under <base>/model/ after every check; raises ValueError (on every rank, before
    any collective call) when there is none or it does not belong to this configuration."""
    path = R.newest_snapshot(os.path.join(args.base_dir, 'model'))
    if path is None:
        raise ValueError('--resume: no snapshot resume-<step>.pt under %s' % os.path.join(args.base_dir, 'model'))
    snap = R.load_snapshot(path)
    R.check_resumable(snap, config_text, n_env)
    return path, snap


def _keep_one_ini(data_dir, name, config_text):
    """A resumed run: data/<name> holds the configuration text it runs (written under a temporary name and renamed, so
    that resuming from the .ini stored in data/ itself is safe), and every other .ini under data/ goes, so that
    evaluate finds this one."""
    tmp = os.path.join(data_dir, '.%s.%d.tmp' % (name, os.getpid()))
    with open(tmp, 'w') as f:
        f.write(config_text)
    os.replace(tmp, os.path.join(data_dir, name))
    for f in os.listdir(data_dir):
        if f.endswith('.ini') and f != name:
            os.remove(os.path.join(data_dir, f))


def train(args):
    world, rank, _ = D.launch_world()
    cfg = read_config(args.config_dir)
    with open(args.config_dir) as f:
        config_text = f.read()
    n_env = cfg.getint('ENV_CONFIG', 'n_env', fallback=1)
    interval = int(cfg.getfloat('TRAIN_CONFIG', 'checkpoint_interval', fallback=0))
    resume = args.resume
    shard = backend = snap = None
    # refused on every rank before the process group exists
    if world > 1:
        shard = D.env_shard(n_env, world, rank)
    if (resume or interval) and n_env == 1:
        raise ValueError('--resume and TRAIN_CONFIG.checkpoint_interval need batched training (ENV_CONFIG.n_env > 1); '
                         'the one-env Trainer cannot be resumed')
    if resume:
        snap_path, snap = _resume_state(args, config_text, n_env)
    if world > 1:
        backend = D.init_from_env()
    lead = rank == 0                                       # rank 0 alone writes the log, data/ and the checkpoint
    if lead:
        dirs = U.init_dir(args.base_dir)
        U.init_log(dirs['log'])
        if resume:
            _keep_one_ini(dirs['data'], os.path.basename(args.config_dir), config_text)
            logging.info('Training: resume from %s at env step %d' % (snap_path, snap['step']))
        else:
            U.copy_file(args.config_dir, dirs['data'])     # evaluate finds the config next to the results
    else:
        logging.basicConfig(format='%(asctime)s [rank ' + str(rank) + '] %(message)s', level=logging.WARNING)
    steps = {k: int(cfg.getfloat('TRAIN_CONFIG', k)) for k in ('total_step', 'test_interval', 'log_interval')}
    env = init_env(cfg['ENV_CONFIG'], shard=shard)
    logging.info('Training: a dim %r, agent dim: %d' % (env.n_a_ls, env.n_agent))
    shard_kw = {} if shard is None else dict(env0=env.env0, n_env_total=env.n_env_total)
    model = init_agent(env, cfg['MODEL_CONFIG'], steps['total_step'], cfg.getint('ENV_CONFIG', 'seed'), **shard_kw)
    if model is None:
        raise SystemExit(2)
    if world > 1:
        # every rank built its weights from the config seed; a change of the init order must not split them silently
        D.check_replicas({'params': model.engine.params})
        logging.info('Training: %d processes (%s), %d of the %d envs each, tensor-core kernels: %s' % (
            world, backend, env.n_env, env.n_env_total, model.engine.use_tc))
    if shard is not None or env.n_env > 1:
        greedy_test = cfg.getboolean('TRAIN_CONFIG', 'greedy_test', fallback=False)
        tester = U.BatchedEvaluator(cfg['ENV_CONFIG'], model, world=world, rank=rank) if greedy_test else None

        def checkpoint(run, step):                          # rank 0: the two files of a periodic checkpoint
            model.save(dirs['model'], step)
            R.save_snapshot(dirs['model'], step, run, config_text, env.n_env_total)
            R.prune(dirs['model'])
            logging.info('Training: checkpoint and snapshot at env step %d' % step)
        final_step = _train_batched(env, model, steps['total_step'], steps['log_interval'],
                                    U.make_summary_writer(dirs['log']) if lead else None,
                                    dirs['data'] if lead else None, tester, graph=backend != 'gloo',
                                    resume=None if snap is None else snap['run'], checkpoint_interval=interval,
                                    checkpoint=checkpoint)
    else:
        counter = U.Counter(steps['total_step'], steps['test_interval'], steps['log_interval'])
        U.Trainer(env, model, counter, U.make_summary_writer(dirs['log']), output_path=dirs['data']).run()
        final_step = counter.cur_step
    if world > 1:
        D.check_replicas({'params': model.engine.params, 'rmsprop ms': model.engine.ms})
        logging.info('Training: parameters and RMSProp state are bit-identical on all %d ranks' % world)
    if lead:
        logging.info('Training: save final model at step %d ...' % final_step)
        model.save(dirs['model'], final_step)
        if interval:
            R.prune(dirs['model'])
    D.shutdown()


def evaluate_fn(agent_dir, output_dir, seeds, port, demo):
    """Load <agent_dir>/data/*.ini and the newest checkpoint under <agent_dir>/model/, run one recorded episode per seed."""
    if not U.check_dir(agent_dir):
        logging.error('Evaluation: %s does not exist!' % os.path.basename(agent_dir))
        return
    ini = U.find_file(agent_dir + '/data/')
    if not ini:
        return
    cfg = read_config(ini)
    env_cfg = nominal_config(cfg['ENV_CONFIG'])          # evaluation runs the nominal scenario parameters
    env_cfg['n_env'] = '1'
    env = init_env(env_cfg, port=port)
    env.init_test_seeds(seeds)
    model = init_agent(env, cfg['MODEL_CONFIG'], 0, 0)
    if model is None or not model.load(agent_dir + '/model/'):
        return
    if demo or not hasattr(model, 'engine'):
        # --demo writes no files; agents without a device engine run the seeds one at a time
        U.Evaluator(env, model, output_dir, gui=demo).run()
    else:
        U.BatchedEvaluator(env_cfg, model, output_dir).run(seeds)


def evaluate(args):
    if D.launch_world()[0] > 1:
        raise ValueError('main.py evaluate runs in one process (all seeds in one batched pass); start it without torchrun')
    output_dir = None
    if not args.demo:
        dirs = U.init_dir(args.base_dir, pathes=['eva_data', 'eva_log'])
        U.init_log(dirs['eva_log'])
        output_dir = dirs['eva_data']
    logging.info('Evaluation: random seeds: %s' % args.evaluation_seeds)
    seeds = [int(s) for s in args.evaluation_seeds.split(',') if s]
    evaluate_fn(args.base_dir, output_dir, seeds, 1, args.demo)


if __name__ == '__main__':
    cli = parse_args()
    {'train': train, 'evaluate': evaluate}[cli.option](cli)
