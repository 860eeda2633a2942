"""Experiment driver with the reference's command line (``main.py:22-155``).

    python -m ic3net_b200.main --env_name predator_prey --nagents 10 --dim 20 --vision 1 \
        --max_steps 80 --hid_size 128 --ic3net --recurrent --nenvs 8192 --num_epochs 1

Every reference flag is accepted with its meaning; flags of subsystems outside the accelerated
path (``--plot``/visdom, ``--display``/curses) are
parsed and rejected with a clear message.  New flags: ``--nenvs`` (environment slots per GPU),
``--obs_mode`` (index | dense), ``--policy_impl`` (tc | simt | tc_tanh | tc_ff), ``--use_graph``.
Multi-GPU: launch with ``python -m torch.distributed.run --nproc-per-node N -m ic3net_b200.main ...``.
"""
import argparse
import os
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
                             'hand-written kernels of the non-recurrent tanh policies (models.MLP, CommNet / IC3Net '
                             'without --recurrent), or torch autograd recompute')
    parser.add_argument('--batch_boundary', default='reference', choices=['reference', 'cut'],
                        help='run_batch: whole episodes until >= batch_size steps per env slot (reference), or a fixed '
                             'number of lock-steps with open episodes cut at the end')
    parser.add_argument('--use_graph', action='store_true', default=False, help='replay the rollout as a CUDA graph')
    parser.add_argument('--rollout_only', action='store_true', default=False,
                        help='collect batches and statistics without the optimizer step')
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


def save_checkpoint(path, policy_net, log, trainer):
    """main.py:260-265."""
    d = dict(policy_net=policy_net.state_dict(), log=log, trainer=trainer.state_dict())
    with _utils_alias():
        torch.save(d, path)


def load_checkpoint(path, policy_net, log, trainer):
    """main.py:267-272."""
    with _utils_alias():
        d = torch.load(path, weights_only=False)
    policy_net.load_state_dict(d['policy_net'])
    log.update({k: LogField(*v) for k, v in d['log'].items()})
    trainer.load_state_dict(d['trainer'])


def main(argv=None):
    argv = sys.argv[1:] if argv is None else argv
    parser = build_parser()
    init_args_for_env(parser, ['x'] + list(argv))
    args = derive_args(parser.parse_args(argv))

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.set_num_threads(1)                         # README.md:48 (OMP_NUM_THREADS=1); host work is tiny
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        torch.distributed.init_process_group("nccl", device_id=dev)
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
    if args.load:
        load_checkpoint(args.load, policy_net, log, trainer)

    for ep in range(args.num_epochs):
        epoch_begin = time.time()
        stat = dict()
        for n in range(args.epoch_size):
            if args.rollout_only:
                batch, s = trainer.run_batch(ep)
            else:
                s = trainer.train_batch(ep)              # main.py:213: the 0-based epoch drives the TJ curriculum
            merge_stat(s, stat)
        epoch_time = time.time() - epoch_begin
        nsteps = stat.get('num_steps', 0)
        epoch = update_log(log, stat)
        if rank == 0:
            for ln in epoch_lines(epoch, stat, epoch_time):
                print(ln)
            print('steps/s {:.0f}'.format(nsteps / max(epoch_time, 1e-9)))
        if args.save_every and ep and args.save != '' and ep % args.save_every == 0 and rank == 0:
            save_checkpoint(args.save + '_' + str(ep), policy_net, log, trainer)
        if args.save != '' and rank == 0:                # main.py:257-258: every epoch
            save_checkpoint(args.save, policy_net, log, trainer)
    if world > 1:
        torch.distributed.destroy_process_group()
    return 0


if __name__ == '__main__':
    sys.exit(main())
