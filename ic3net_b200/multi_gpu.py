"""Data-parallel trainer: the multi-GPU replacement of the reference's ``multi_processing.py``.

Reference (multi_processing.py:41-104): N forked processes share the parameters, each runs
``run_batch`` + ``compute_grad`` on its own environment, the master sums the per-process
gradients through shared memory, divides by the GLOBAL number of env steps and takes one
RMSprop step (:90-97); ``stat`` dicts are merged with ``merge_stat`` (:86-88).

Here: one process per GPU (``torch.distributed``; NCCL over NVLink on GPUs, gloo in the CPU
tests), parameters replicated, environment slots sharded (rank r owns global env ids
``[r*B, (r+1)*B)``, i.e. ``args.env_id0 = rank * args.nenvs`` selects its Philox streams).
The reference's workers share ONE set of parameters (main.py:177-179 ``share_memory_``); the
replicas get the same guarantee from a broadcast of rank 0's flat parameter (and optimizer
state) buffer at construction and after ``load_state_dict``.  Per update exactly ONE gradient
collective: an all-reduce(sum) of the flat fp32 gradient buffer (parameters without a gradient
-- ``hidd_encoder`` -- are skipped like multi_processing.py:35,65), then ``grad /= global
num_steps`` and the same optimizer step on every rank, so the replicas stay bit-identical.  The
batch statistics and the loss sums never leave the device before they are reduced: they ride a
second, ~200-byte float64 all-reduce (step / episode counts stay exact) and reach the host in
ONE copy per update.
"""
import numbers

import numpy as np
import torch
import torch.distributed as dist

from .trainer import check_fingerprint
from .utils import merge_stat


def _dist_on():
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def flat_grad_buffer(params):
    """One contiguous fp32 buffer holding every existing gradient (in parameter order)."""
    gs = [p.grad for p in params if p.grad is not None]
    if not gs:
        return None, []
    flat = torch.cat([g.reshape(-1) for g in gs])
    return flat, gs


def unflatten_into(flat, grads):
    off = 0
    for g in grads:
        n = g.numel()
        g.copy_(flat[off:off + n].view_as(g))
        off += n


def pack_stat(stat, device):
    """Numbers and numpy arrays (merge_stat's additive kinds, utils.py:19-22) -> float64 vector."""
    keys = sorted(k for k, v in stat.items() if isinstance(v, (numbers.Number, np.ndarray)))
    parts, shapes = [], []
    for k in keys:
        v = np.atleast_1d(np.asarray(stat[k], dtype=np.float64))
        shapes.append((k, v.shape, isinstance(stat[k], numbers.Number)))
        parts.append(v.ravel())
    vec = torch.from_numpy(np.concatenate(parts) if parts else np.zeros(0)).to(device)
    return vec, shapes


def unpack_stat(vec, shapes, stat):
    v = vec.cpu().numpy()
    off = 0
    for k, shp, scalar in shapes:
        n = int(np.prod(shp))
        x = v[off:off + n].reshape(shp)
        off += n
        if scalar:
            x = float(x[0])
            stat[k] = int(round(x)) if abs(x - round(x)) < 1e-9 else x
        else:
            stat[k] = x
    return stat


class MultiGPUTrainer(object):
    """Same surface as ``MultiProcessTrainer``: ``train_batch``, ``quit``, ``state_dict``,
    ``load_state_dict`` (multi_processing.py:41-104)."""

    def __init__(self, args, trainer_maker):
        self.args = args
        self.trainer = trainer_maker()
        self.world = dist.get_world_size() if _dist_on() else 1
        self.rank = dist.get_rank() if _dist_on() else 0
        self.is_random = getattr(args, 'random', False)
        self.collectives = 0          # gradient all-reduces issued (one per update)
        self.sync_parameters()

    def quit(self):
        return

    # ------------------------------------------------------------------ replicas
    def sync_parameters(self):
        """Every rank takes rank 0's parameters and optimizer state (the reference's workers share one policy,
        main.py:177-179).  A no-op for a single process."""
        if not _dist_on():
            return
        opt = self.trainer.optimizer
        if hasattr(opt, 'flat_params'):
            dist.broadcast(opt.flat_params, src=0)
            dist.broadcast(opt.flat_square_avg, src=0)
            steps = torch.tensor([opt.steps], dtype=torch.int64, device=opt.flat_params.device)
            dist.broadcast(steps, src=0)
            opt.steps = int(steps.item())
            opt.mark_params_changed()
        else:
            for p in self.trainer.params:
                dist.broadcast(p.data, src=0)

    def replica_checksum(self):
        """(max |param - rank 0's param|) over all ranks; 0.0 when the replicas are bit-identical."""
        opt = self.trainer.optimizer
        flat = opt.flat_params if hasattr(opt, 'flat_params') else torch.cat([p.data.reshape(-1) for p in self.trainer.params])
        if not _dist_on():
            return 0.0
        ref = flat.clone()
        dist.broadcast(ref, src=0)
        d = (flat - ref).abs().max().reshape(1)
        dist.all_reduce(d, op=dist.ReduceOp.MAX)
        return float(d.item())

    # ------------------------------------------------------------------ reductions
    def reduce(self, stat):
        """Sum gradients and additive stats (a HOST dict) over ranks; returns the merged stat.  Generic path
        (any trainer with ``params`` / ``optimizer``); Trainer.update avoids the host dict."""
        params = self.trainer.params
        opt = self.trainer.optimizer
        if hasattr(opt, 'flat_grads'):
            # FlatRMSprop: the gradients already live in one buffer -> all-reduce it in place; the division by the
            # global step count (multi_processing.py:95) is folded into the optimizer kernel (train_batch below)
            vec, shapes = pack_stat(stat, opt.flat_grads.device)
            if _dist_on():
                dist.all_reduce(opt.flat_grads, op=dist.ReduceOp.SUM)      # multi_processing.py:92-94
                self.collectives += 1
                dist.all_reduce(vec, op=dist.ReduceOp.SUM)                 # multi_processing.py:86-88
            return unpack_stat(vec, shapes, dict(stat))
        flat, grads = flat_grad_buffer(params)
        dev = flat.device if flat is not None else (params[0].device if params else torch.device('cpu'))
        vec, shapes = pack_stat(stat, dev)
        if _dist_on():
            if flat is not None:
                dist.all_reduce(flat, op=dist.ReduceOp.SUM)      # multi_processing.py:92-94
                self.collectives += 1
            dist.all_reduce(vec, op=dist.ReduceOp.SUM)           # multi_processing.py:86-88
        stat = unpack_stat(vec, shapes, dict(stat))
        if flat is not None:
            flat /= stat['num_steps']                            # multi_processing.py:95 (global step count)
            unflatten_into(flat, grads)
        return stat

    def reduce_device(self, loss_vec=None, with_grads=True):
        """Device path: all-reduce the flat gradient buffer (in place) and the float64 [batch statistics | loss
        sums] vector, then ONE device->host copy.  Returns the merged stat dict of all ranks."""
        tr = self.trainer
        vec = tr.stat_vector()
        nstat = vec.numel()
        if loss_vec is not None:
            vec = torch.cat([vec, loss_vec.to(vec.dtype)])
        if _dist_on():
            if with_grads:
                dist.all_reduce(tr.optimizer.flat_grads, op=dist.ReduceOp.SUM)     # multi_processing.py:92-94
                self.collectives += 1
            dist.all_reduce(vec, op=dist.ReduceOp.SUM)                             # multi_processing.py:86-88
        host = vec.cpu().numpy()
        stat = tr.stat_from_vector(host[:nstat])
        if loss_vec is not None:
            for i, k in enumerate(tr.LOSS_KEYS):
                stat[k] = float(host[nstat + i])
        return stat

    def _reduce_in_place(self, vec):
        """Trainer.update's reduce: all-reduce(sum) the flat gradient buffer (not for models.Random, which has no
        gradient) and the device vector [statistics | loss sums | ...] in place (multi_processing.py:86-94)."""
        if not self.trainer.random_policy:
            dist.all_reduce(self.trainer.optimizer.flat_grads, op=dist.ReduceOp.SUM)
            self.collectives += 1
        dist.all_reduce(vec, op=dist.ReduceOp.SUM)

    def run_batch(self, epoch):
        """Rollout only (``--rollout_only``): every rank collects its batch; statistics merged over ranks."""
        tr = self.trainer
        T, quota = tr.batch_plan()
        batch = tr.rollout(T, epoch, quota=quota)
        return batch, self.reduce_device(None, with_grads=False)

    def train_batch(self, epoch):
        tr = self.trainer
        if hasattr(tr, 'update'):
            # the reduce runs between the head (rollout .. gradients) and the tail (optimizer step, weight pack), eagerly
            # also when graph_update replays both: NCCL calls stay outside any capture
            return tr.update(epoch, self._reduce_in_place if _dist_on() else None)
        batch, stat = tr.run_batch(epoch)
        tr.optimizer.zero_grad(set_to_none=False)
        s = tr.compute_grad(batch)
        merge_stat(s, stat)
        stat = self.reduce(stat)
        if hasattr(tr.optimizer, 'flat_grads'):
            tr.optimizer.step(grad_div=stat['num_steps'])        # multi_processing.py:95-97 in one kernel
        else:
            tr.optimizer.step()                                  # multi_processing.py:97
        return stat

    def evaluate(self, episodes=1, greedy=False, epoch=None):
        """Trainer.evaluate on every rank's evaluation slots; the statistics vector is summed over ranks with one
        all-reduce, so every rank returns the stat dict of all ranks' episodes."""
        tr = self.trainer
        vec, e = tr.evaluate_vector(episodes, greedy, epoch)
        if _dist_on():
            dist.all_reduce(vec, op=dist.ReduceOp.SUM)
        return tr.stat_from_vector(vec.cpu().numpy(), e)

    def evaluate_trace(self, episodes=1, greedy=False, epoch=None, slots=8, comm_map=True, messages=False):
        """Trainer.evaluate_trace on every rank's evaluation slots: the statistics vector, the comm map and the message
        map's integer sums are summed over ranks (one all-reduce each, exact), the trace is of this rank's slots (its
        env_id holds their global ids)."""
        tr = self.trainer
        vec, e, rec = tr.evaluate_trace_vector(episodes, greedy, epoch, slots, comm_map, messages)
        if _dist_on():
            dist.all_reduce(vec, op=dist.ReduceOp.SUM)
            if rec.counts is not None:
                dist.all_reduce(rec.counts, op=dist.ReduceOp.SUM)
            if rec.msg_sums is not None:
                dist.all_reduce(rec.msg_sums, op=dist.ReduceOp.SUM)
        stat = tr.stat_from_vector(vec.cpu().numpy(), e)
        trace, cmap = rec.to_host()
        return stat, trace, cmap

    def state_dict(self):
        return self.trainer.state_dict()

    def load_state_dict(self, state):
        self.trainer.load_state_dict(state)
        self.sync_parameters()

    def run_state(self):
        """Trainer.run_state over every rank: each rank's state is gathered to rank 0, which returns
        {'fingerprint', 'ranks': [rank 0's, rank 1's, ...]}; the other ranks return None.  Every rank must call it."""
        tr = self.trainer
        if not _dist_on():
            return tr.run_state()
        mine = tr.rank_state()
        got = [None] * self.world if self.rank == 0 else None
        dist.gather_object(mine, got, dst=0)
        return dict(fingerprint=tr.run_fingerprint(), ranks=got) if self.rank == 0 else None

    def load_run_state(self, state):
        """Every rank loads the same state (written by rank 0) and takes its own slice; the fingerprint, world size
        included, must match."""
        check_fingerprint(state['fingerprint'], self.trainer.run_fingerprint())
        self.trainer.load_rank_state(state['ranks'][self.rank])
