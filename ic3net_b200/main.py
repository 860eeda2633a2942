"""Experiment driver with the reference's command line (``main.py:22-155``).

    python -m ic3net_b200.main --env_name predator_prey --nagents 10 --dim 20 --vision 1 \
        --max_steps 80 --hid_size 128 --ic3net --recurrent --nenvs 8192 --num_epochs 1

Every reference flag is accepted with its meaning; flags of subsystems outside the accelerated
path (``--plot``/visdom, ``--display``/curses) are
parsed and rejected with a clear message.  New flags: ``--nenvs`` (environment slots per GPU),
``--obs_mode`` (index | dense), ``--policy_impl`` (tc | simt | tc_tanh | tc_ff), ``--use_graph``, ``--graph_update``,
and evaluation of whole episodes every K epochs (``--eval_every``, ``--eval_episodes``, ``--eval_nenvs``,
``--eval_greedy``; Trainer.evaluate), and resuming an interrupted run exactly where it stopped (``--resumable``,
``--resume``: a run-state sidecar beside every checkpoint; SIGTERM / SIGINT save and exit after the update in flight).
Multi-GPU: launch with ``python -m torch.distributed.run --nproc-per-node N -m ic3net_b200.main ...``.
"""
import argparse
import os
import signal
import sys
import time

import numpy as np
import torch

from . import data
from .action_utils import parse_action_args
from .comm import CommNetMLP
from .multi_gpu import MultiGPUTrainer
from .trainer import Trainer
from .utils import LogField, init_args_for_env, merge_stat


def build_parser():
    parser = argparse.ArgumentParser(description='PyTorch RL trainer (GPU rollout path)')
    # training (main.py:24-31)
    parser.add_argument('--num_epochs', default=100, type=int, help='number of training epochs')
    parser.add_argument('--epoch_size', type=int, default=10, help='number of update iterations in an epoch')
    parser.add_argument('--batch_size', type=int, default=500, help='number of steps before each update (per env slot)')
    parser.add_argument('--nprocesses', type=int, default=16, help='kept for compatibility; ranks come from torchrun')
    # model (main.py:33-36)
    parser.add_argument('--hid_size', default=64, type=int, help='hidden layer size')
    parser.add_argument('--recurrent', action='store_true', default=False, help='make the model recurrent in time')
    # optimization (main.py:38-52)
    parser.add_argument('--gamma', type=float, default=1.0, help='discount factor')
    parser.add_argument('--tau', type=float, default=1.0, help='gae (remove?)')
    parser.add_argument('--seed', type=int, default=-1, help='random seed. Pass -1 for random seed')
    parser.add_argument('--normalize_rewards', action='store_true', default=False, help='normalize rewards in each batch')
    parser.add_argument('--lrate', type=float, default=0.001, help='learning rate')
    parser.add_argument('--entr', type=float, default=0, help='entropy regularization coeff')
    parser.add_argument('--value_coeff', type=float, default=0.01, help='coeff for value loss term')
    # environment (main.py:54-61)
    parser.add_argument('--env_name', default="Cartpole", help='name of the environment to run')
    parser.add_argument('--max_steps', default=20, type=int, help='force to end the game after this many steps')
    parser.add_argument('--nactions', default='1', type=str, help='the number of agent actions')
    parser.add_argument('--action_scale', default=1.0, type=float, help='scale action output from model')
    # other (main.py:63-78)
    parser.add_argument('--plot', action='store_true', default=False, help='plot training progress')
    parser.add_argument('--plot_env', default='main', type=str, help='plot env name')
    parser.add_argument('--save', default='', type=str, help='save the model after training')
    parser.add_argument('--save_every', default=0, type=int, help='save the model after every n_th epoch')
    parser.add_argument('--load', default='', type=str, help='load the model')
    parser.add_argument('--display', action="store_true", default=False, help='Display environment state')
    parser.add_argument('--random', action='store_true', default=False, help="enable random model")
    # CommNet specific args (main.py:81-109)
    parser.add_argument('--commnet', action='store_true', default=False, help="enable commnet model")
    parser.add_argument('--ic3net', action='store_true', default=False, help="enable commnet model")
    parser.add_argument('--nagents', type=int, default=1, help="Number of agents (used in multiagent)")
    parser.add_argument('--comm_mode', type=str, default='avg', help="[avg|sum]")
    parser.add_argument('--comm_passes', type=int, default=1, help="Number of comm passes per step over the model")
    parser.add_argument('--comm_mask_zero', action='store_true', default=False, help="Whether communication should be there")
    parser.add_argument('--mean_ratio', default=1.0, type=float, help='how much coooperative to do? 1.0 means fully cooperative')
    parser.add_argument('--rnn_type', default='MLP', type=str, help='type of rnn to use. [LSTM|MLP]')
    parser.add_argument('--detach_gap', default=10000, type=int, help='detach hidden state and cell state at this interval')
    parser.add_argument('--comm_init', default='uniform', type=str, help='how to initialise comm weights [uniform|zeros]')
    parser.add_argument('--hard_attn', default=False, action='store_true', help='hard attention: action - talk|silent')
    parser.add_argument('--comm_action_one', default=False, action='store_true', help='always talk')
    parser.add_argument('--advantages_per_action', default=False, action='store_true',
                        help='accepted; the per-head products of trainer.py:189-199 sum to the same loss and gradient '
                             '(tests/test_host_logic.py pins that on the reference), so there is one code path')
    parser.add_argument('--share_weights', default=False, action='store_true', help='Share weights for hops')
    # additions of the GPU rollout path
    parser.add_argument('--nenvs', type=int, default=1024, help='environment slots per GPU')
    parser.add_argument('--obs_mode', default='index', choices=['index', 'dense'],
                        help='encoder fed from the env state (index) or from a materialised [B,N,O] observation (dense)')
    parser.add_argument('--obs_api', default='dense', choices=['dense', 'handle'],
                        help='what env.reset/step hand back: the dense [nenvs,N,obs_dim] tensor, or a LazyObs handle on the '
                             'env state that CommNetMLP.forward consumes directly (lazy_obs.py)')
    parser.add_argument('--policy_impl', default=None, choices=['tc', 'simt', 'tc_tanh', 'tc_ff'],
                        help='wgmma tensor-core or fp32 SIMT policy kernels; tc_tanh: the tensor-core step of the '
                             'tanh RNN (IC / IRIC: --recurrent without --commnet, hid_size 128); tc_ff: the tensor-core '
                             'step of the non-recurrent tanh policies (MLP, CommNet / IC3Net without --recurrent, '
                             'hid_size 128)')
    parser.add_argument('--grad_impl', default='auto', choices=['auto', 'kernels', 'kernels_ff', 'autograd'],
                        help='compute_grad: hand-written BPTT kernels (auto: whenever the configuration allows), the '
                             'hand-written tensor-core kernels of the non-recurrent tanh policies (kernels_ff: '
                             'models.MLP, CommNet / IC3Net without --recurrent), or torch autograd recompute')
    parser.add_argument('--batch_boundary', default='reference', choices=['reference', 'cut'],
                        help='run_batch: whole episodes until >= batch_size steps per env slot (reference), or a fixed '
                             'number of lock-steps with open episodes cut at the end')
    parser.add_argument('--use_graph', action='store_true', default=False, help='replay the rollout as a CUDA graph')
    parser.add_argument('--graph_update', action='store_true', default=False,
                        help='replay each whole training update (rollout, gradient kernels, RMSprop, weight pack) from '
                             'CUDA graphs with one host read per update; needs grad_impl kernels or kernels_ff')
    parser.add_argument('--rollout_only', action='store_true', default=False,
                        help='collect batches and statistics without the optimizer step')
    parser.add_argument('--eval_every', type=int, default=0,
                        help='evaluate the policy every K epochs on whole episodes (0: never)')
    parser.add_argument('--eval_episodes', type=int, default=1, help='episodes per evaluation slot')
    parser.add_argument('--eval_nenvs', type=int, default=None, help='evaluation slots per GPU (default: --nenvs)')
    parser.add_argument('--eval_greedy', action='store_true', default=False,
                        help='evaluate with the argmax action of every head instead of sampled actions')
    parser.add_argument('--eval_trace', type=str, default='',
                        help='with --eval_every: record every evaluation and write PREFIX_epoch<E>.npz (rank 0\'s slots: '
                             'per-step trajectories and the map of where agents open their gate)')
    parser.add_argument('--eval_trace_slots', type=int, default=8, help='evaluation slots recorded by --eval_trace')
    parser.add_argument('--eval_trace_messages', action='store_true', default=False,
                        help='with --eval_trace: also record what the agents communicate (recurrent CommNet / IC3Net, '
                             'one comm pass): the hidden state each sends, its gate and the vector it receives, and '
                             'their sums by cell and episode step (msg_* and map_msg_* arrays)')
    parser.add_argument('--resumable', action='store_true', default=False,
                        help='with --save: every checkpoint write also writes the run state to <checkpoint>.run, and '
                             'SIGTERM / SIGINT save both and exit after the update in flight, so --resume can continue '
                             'the run bit for bit')
    parser.add_argument('--resume', default='', type=str,
                        help='continue the run saved with --resumable at checkpoint PATH (and PATH.run) at the epoch '
                             'and update where it stopped; --num_epochs stays the total of the whole run')
    return parser


def derive_args(args):
    """main.py:115-155."""
    if args.ic3net:
        args.commnet = 1
        args.hard_attn = 1
        args.mean_ratio = 0
        if args.env_name == "traffic_junction":
            args.comm_action_one = True
    args.nfriendly = args.nagents
    if getattr(args, 'enemy_comm', False):       # main.py:126-130: the enemies become agents of the policy
        if hasattr(args, 'nenemies'):
            args.nagents += args.nenemies
        else:
            raise RuntimeError("Env. needs to pass argument 'nenemy'.")
    if args.plot or args.display:
        raise NotImplementedError("--plot / --display (visdom, curses) are outside the accelerated path")
    return args


def make_policy(args, num_inputs):
    """main.py:162-169."""
    from . import models
    if args.commnet:
        return CommNetMLP(args, num_inputs)
    if args.random:
        return models.Random(args, num_inputs)
    if args.recurrent:
        return models.RNN(args, num_inputs)
    return models.MLP(args, num_inputs)


LOG_FIELDS = (('epoch', None), ('reward', 'num_episodes'), ('enemy_reward', 'num_episodes'),
              ('success', 'num_episodes'), ('steps_taken', 'num_episodes'), ('add_rate', 'num_episodes'),
              ('comm_action', 'num_steps'), ('enemy_comm', 'num_steps'), ('value_loss', 'num_steps'),
              ('action_loss', 'num_steps'), ('entropy', 'num_steps'))


def make_log():
    """The reference's log table (main.py:194-205): same keys, plot flags, x axes and divisors."""
    log = dict()
    for k, d in LOG_FIELDS:
        log[k] = LogField(list(), k != 'epoch', 'epoch' if k != 'epoch' else None, d)
    return log


def update_log(log, stat):
    """End-of-epoch bookkeeping with the reference's contract (main.py:218-225), in place on both arguments.
    The merged ``stat`` of the epoch is normalised field by field -- a field that has a divisor (``num_episodes`` or
    ``num_steps``) is divided by it when that count is positive -- and EVERY series of the log receives exactly one
    entry per epoch (0 for a field the epoch did not produce), so all series stay aligned with ``log['epoch']``.
    Returns the 1-based epoch number."""
    epoch = len(log['epoch'].data) + 1
    log['epoch'].data.append(epoch)
    for name, field in log.items():
        if name == 'epoch':
            continue
        div = field.divide_by
        if name in stat and div is not None and stat[div] > 0:
            stat[name] = stat[name] / stat[div]
        field.data.append(stat.get(name, 0))
    return epoch


# (stat key, line format) in the order the reference prints them (main.py:233-244)
_EPOCH_LINES = (('enemy_reward', 'Enemy-Reward: {}'), ('add_rate', 'Add-Rate: {:.2f}'), ('success', 'Success: {:.2f}'),
                ('steps_taken', 'Steps-taken: {:.2f}'), ('comm_action', 'Comm-Action: {}'),
                ('enemy_comm', 'Enemy-Comm: {}'))


def epoch_lines(epoch, stat, epoch_time):
    """What main.py:227-244 prints for an epoch, as a list of lines (``stat`` already normalised by update_log)."""
    np.set_printoptions(precision=2)
    head = 'Epoch {}\tReward {}\tTime {:.2f}s'.format(epoch, stat['reward'], epoch_time)
    return [head] + [fmt.format(stat[key]) for key, fmt in _EPOCH_LINES if key in stat]


def eval_line(stat, greedy, episodes, slots):
    """The line printed for an evaluation: its stat dict (raw sums, Trainer.evaluate) normalised field by field as
    update_log normalises an epoch's, without touching the log."""
    np.set_printoptions(precision=2)
    div = dict(LOG_FIELDS)
    v = {k: (stat[k] / stat[div[k]] if div.get(k) and stat[div[k]] > 0 else stat[k]) for k in stat}
    parts = [fmt.format(v[k]) for k, fmt in (('success', 'Success {:.2f}'), ('reward', 'Reward {}'),
                                             ('steps_taken', 'Steps-taken {:.2f}'), ('comm_action', 'Comm-Action {}'))
             if k in v]
    return 'Eval ({}, {} episodes \u00d7 {} slots): '.format('greedy' if greedy else 'sampled', episodes, slots) + \
        '  '.join(parts)


class _utils_alias(object):
    """Checkpoints interchange with the reference (main.py:260-272): its ``log`` is pickled as ``utils.LogField``.
    Inside this context the name ``utils`` resolves to ic3net_b200.utils and our LogField class pickles under that name, so files written here load in the reference and
    files written by the reference load here."""

    def __enter__(self):
        from . import utils as _u
        self._had = sys.modules.get('utils')
        sys.modules['utils'] = _u
        self._mod = LogField.__module__
        LogField.__module__ = 'utils'
        return self

    def __exit__(self, *e):
        LogField.__module__ = self._mod
        if self._had is None:
            sys.modules.pop('utils', None)
        else:
            sys.modules['utils'] = self._had
        return False


def write_atomic(writers):
    """writers: [(path, write(tmp_path))].  Every file is written under a temporary name beside its path first, then
    all are moved into place with os.replace.  If a writer fails, its temporaries are removed and the files already
    at the paths stay as they were."""
    tmps = []
    try:
        for path, write in writers:
            tmps.append('%s.tmp%d' % (path, os.getpid()))
            write(tmps[-1])
    except BaseException:
        for t in tmps:
            if os.path.exists(t):
                os.remove(t)
        raise
    for (path, _), t in zip(writers, tmps):
        os.replace(t, path)


def checkpoint_position(d):
    """(optimizer steps, logged epochs) of a checkpoint dict: a run-state sidecar records both, so a sidecar that
    does not belong to its checkpoint (a kill between the two renames of a save) is recognised."""
    steps = [int(float(st.get('step', 0))) for st in d['trainer']['state'].values()]
    return max(steps, default=0), len(d['log']['epoch'].data)


def save_checkpoint(path, policy_net, log, trainer, evals=None, run=None):
    """main.py:260-265; evals: the evaluation results [(epoch, stat dict)], stored under 'eval' unless None.
    run: with --resumable, {'ep', 'update', 'stat', 'state'} -- the loop position (the 0-based epoch, the updates of
    it done, their merged stat) and the trainer's run_state() -- written to path + '.run' beside the checkpoint, with
    the checkpoint's optimizer steps and epochs.  Both files are replaced atomically (write_atomic)."""
    d = dict(policy_net=policy_net.state_dict(), log=log, trainer=trainer.state_dict())
    if evals is not None:
        d['eval'] = list(evals)

    def write(p):
        with _utils_alias():
            torch.save(d, p)
    writers = [(path, write)]
    if run is not None:
        steps, epochs = checkpoint_position(d)
        side = dict(run, version=RUN_FILE_VERSION, steps=steps, epochs=epochs)
        writers.append((path + '.run', lambda p: torch.save(side, p)))
    write_atomic(writers)


RUN_FILE_VERSION = 1


def read_run_file(path):
    """The run-state sidecar of checkpoint path (save_checkpoint's ``run``, plus 'version', 'steps', 'epochs')."""
    if not os.path.exists(path + '.run'):
        raise FileNotFoundError("no run state %s.run beside the checkpoint %s: --resume continues a run saved with "
                                "--resumable (--load restores the policy and log of any checkpoint)" % (path, path))
    run = torch.load(path + '.run', weights_only=False)
    if run.get('version') != RUN_FILE_VERSION:
        raise ValueError("%s.run has version %r; this program reads version %d" % (path, run.get('version'),
                                                                                  RUN_FILE_VERSION))
    return run


def save_eval_trace(prefix, epoch, args, grid_shape, trace, cmap):
    """PREFIX_epoch<E>.npz: the trace's arrays, the comm map's (and the message map's) under 'map_<key>', and what it
    takes to read them (with messages also hid_size)."""
    d = dict(trace.arrays())
    for k, v in (cmap or {}).items():
        d['map_' + k] = v
    pp = args.env_name == 'predator_prey'
    d.update(env_name=np.array(args.env_name), grid_shape=np.asarray(grid_shape, dtype=np.int64),
             nagents=np.int64(args.nagents),
             nfriendly=np.int64(getattr(args, 'nfriendly', args.nagents) if pp else args.nagents),
             naction_heads=np.asarray(args.naction_heads, dtype=np.int64), max_steps=np.int64(args.max_steps),
             episodes=np.int64(args.eval_episodes), greedy=np.int64(bool(args.eval_greedy)),
             hard_attn=np.int64(bool(args.hard_attn and args.commnet)))
    if trace.msg_h is not None:
        d['hid_size'] = np.int64(args.hid_size)
    np.savez(prefix + '_epoch%d.npz' % epoch, **d)


def load_checkpoint(path, policy_net, log, trainer):
    """main.py:267-272.  Returns the checkpoint's evaluation results [(epoch, stat dict)] ([] without 'eval')."""
    with _utils_alias():
        d = torch.load(path, weights_only=False)
    return _apply_checkpoint(d, policy_net, log, trainer)


def _apply_checkpoint(d, policy_net, log, trainer):
    policy_net.load_state_dict(d['policy_net'])
    log.update({k: LogField(*v) for k, v in d['log'].items()})
    trainer.load_state_dict(d['trainer'])
    return list(d.get('eval', []))


def resume_checkpoint(path, run, policy_net, log, trainer):
    """--resume: load_checkpoint after checking that run (read_run_file) belongs to the checkpoint and loading its run
    state into the trainer (which refuses another configuration).  Returns the checkpoint's evaluation results."""
    with _utils_alias():
        d = torch.load(path, weights_only=False)
    have = checkpoint_position(d)
    if have != (run['steps'], run['epochs']):
        raise ValueError("%s.run does not belong to %s: it was written after %d optimizer steps and %d epochs, the "
                         "checkpoint after %d and %d (a save was interrupted between its two files)"
                         % (path, path, run['steps'], run['epochs'], have[0], have[1]))
    trainer.load_run_state(run['state'])
    return _apply_checkpoint(d, policy_net, log, trainer)


class StopOnSignal(object):
    """--resumable: SIGTERM and SIGINT only raise a flag; the training loop saves and exits after the update in flight.
    restore() puts the previous handlers back."""
    SIGNALS = (signal.SIGTERM, signal.SIGINT)

    def __init__(self):
        self.raised = False
        self._old = {s: signal.signal(s, self._raise) for s in self.SIGNALS}

    def _raise(self, signum, frame):
        self.raised = True

    def restore(self):
        for s, h in self._old.items():
            signal.signal(s, h)

    def agreed(self, device, world):
        """Has any rank been signalled?  A signal can reach the ranks at different updates, so they agree through a
        one-element all-reduce (MAX) after every update."""
        if world == 1:
            return self.raised
        f = torch.tensor([int(self.raised)], dtype=torch.int32, device=device)
        torch.distributed.all_reduce(f, op=torch.distributed.ReduceOp.MAX)
        return bool(f.item())


def main(argv=None):
    argv = sys.argv[1:] if argv is None else argv
    parser = build_parser()
    init_args_for_env(parser, ['x'] + list(argv))
    args = derive_args(parser.parse_args(argv))
    if args.resume and args.load:
        parser.error("--resume continues a run from its checkpoint and run state; it takes no --load")
    if args.resumable and not args.save:
        parser.error("--resumable writes the run state beside the --save checkpoint; give --save")
    if args.eval_trace_messages and not args.eval_trace:
        parser.error("--eval_trace_messages adds to the recording of --eval_trace; give --eval_trace")
    run = read_run_file(args.resume) if args.resume else None
    args.resumable = args.resumable or bool(args.resume and args.save)

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.set_num_threads(1)                         # README.md:48 (OMP_NUM_THREADS=1); host work is tiny
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        torch.distributed.init_process_group("nccl", device_id=dev)
    if run is not None and args.seed == -1:          # a resumed run plays on the streams of the run it continues
        args.seed = int(run['state']['fingerprint']['seed'])
    if args.seed == -1:                              # main.py:157-158; ONE draw for the whole job: rank 0's
        seed = torch.tensor([int(np.random.randint(0, 10000))], dtype=torch.int64, device=dev)
        if world > 1:
            torch.distributed.broadcast(seed, src=0)
        args.seed = int(seed.item())
    args.env_id0 = rank * args.nenvs                 # this rank's slice of the global env ids
    torch.manual_seed(args.seed)                     # identical initial parameters on every rank (main.py:159)

    env = data.init(args.env_name, args, False)
    num_inputs = env.observation_dim
    args.num_actions = env.num_actions
    if not isinstance(args.num_actions, (list, tuple)):
        args.num_actions = [args.num_actions]
    args.dim_actions = env.dim_actions
    args.num_inputs = num_inputs
    if args.hard_attn and args.commnet:
        args.num_actions = [*args.num_actions, 2]
        args.dim_actions = env.dim_actions + 1
    if args.commnet and (args.recurrent or args.rnn_type == 'LSTM'):
        args.recurrent = True
        args.rnn_type = 'LSTM'
    parse_action_args(args)
    if rank == 0:
        print(args)

    args.record_for_grad = not args.rollout_only     # keep the inputs compute_grad re-runs (trainer.py)
    policy_net = make_policy(args, num_inputs)
    # MultiGPUTrainer broadcasts rank 0's parameters: replicas are identical whatever the ranks' RNG state was
    trainer = MultiGPUTrainer(args, lambda: Trainer(args, policy_net, env))

    log = make_log()
    evals = []
    if args.load:
        evals = load_checkpoint(args.load, policy_net, log, trainer)
    start_ep, start_update, partial = 0, 0, None
    if run is not None:
        evals = resume_checkpoint(args.resume, run, policy_net, log, trainer)
        start_ep, start_update, partial = run['ep'], run['update'], run['stat']
    eval_slots = world * (args.eval_nenvs or args.nenvs)
    stop = StopOnSignal() if args.resumable else None
    try:
        _train(args, trainer, policy_net, env, log, evals, eval_slots, rank, world, dev, stop, start_ep, start_update,
               partial)
    finally:
        if stop is not None:
            stop.restore()
    if world > 1:
        torch.distributed.destroy_process_group()
    return 0


def _train(args, trainer, policy_net, env, log, evals, eval_slots, rank, world, dev, stop, start_ep, start_update,
           partial):
    """The epoch loop of main.py:207-258 from epoch start_ep, update start_update, with the merged stat partial of the
    updates of that epoch already done (a resumed run)."""
    for ep in range(start_ep, args.num_epochs):
        epoch_begin = time.time()
        first = ep == start_ep
        stat = dict(partial) if first and partial else dict()
        for n in range(start_update if first else 0, args.epoch_size):
            if args.rollout_only:
                batch, s = trainer.run_batch(ep)
            else:
                s = trainer.train_batch(ep)              # main.py:213: the 0-based epoch drives the TJ curriculum
            merge_stat(s, stat)
            if stop is not None and stop.agreed(dev, world):
                state = trainer.run_state()              # gathered from every rank
                if rank == 0:
                    save_checkpoint(args.save, policy_net, log, trainer, evals if (evals or args.eval_every) else None,
                                    dict(ep=ep, update=n + 1, stat=stat, state=state))
                    print('Stopped in epoch {} after update {} of {}; continue with --resume {}'.format(
                        ep + 1, n + 1, args.epoch_size, args.save), flush=True)
                return
        epoch_time = time.time() - epoch_begin
        nsteps = stat.get('num_steps', 0)
        epoch = update_log(log, stat)
        if rank == 0:
            for ln in epoch_lines(epoch, stat, epoch_time):
                print(ln)
            print('steps/s {:.0f}'.format(nsteps / max(epoch_time, 1e-9)))
        if args.eval_every and epoch % args.eval_every == 0:    # every rank plays its slots; the sum is reduced
            if args.eval_trace:
                cfg, tj = env.env.cfg, args.env_name == 'traffic_junction'
                es, trace, cmap = trainer.evaluate_trace(args.eval_episodes, args.eval_greedy,
                                                         slots=min(args.eval_trace_slots, args.eval_nenvs or args.nenvs),
                                                         messages=args.eval_trace_messages)
                if rank == 0:
                    save_eval_trace(args.eval_trace, epoch, args, (cfg.h, cfg.w) if tj else (cfg.dim, cfg.dim),
                                    trace, cmap)
            else:
                es = trainer.evaluate(args.eval_episodes, args.eval_greedy)
            evals.append((epoch, es))
            if rank == 0:
                print(eval_line(es, args.eval_greedy, args.eval_episodes, eval_slots))
        ck = evals if (evals or args.eval_every) else None     # without evaluation the checkpoint stays as it was
        run = dict(ep=ep + 1, update=0, stat=None, state=trainer.run_state()) if args.resumable else None
        if args.save_every and ep and args.save != '' and ep % args.save_every == 0 and rank == 0:
            save_checkpoint(args.save + '_' + str(ep), policy_net, log, trainer, ck, run)
        if args.save != '' and rank == 0:                # main.py:257-258: every epoch
            save_checkpoint(args.save, policy_net, log, trainer, ck, run)


if __name__ == '__main__':
    sys.exit(main())
