"""Batched GPU rollout + REINFORCE gradient behind the reference's ``trainer.Trainer`` surface
(trainer.py:14-262).

``Trainer(args, policy_net, env)`` drives ``env.nenvs`` independent environment slots in
lock-step on one GPU.  Each slot plays the role of one reference process: it runs episode after
episode (auto-reset, hidden state zeroed, nobody talks at t = 0), and ``run_batch`` follows the
reference's batch boundary (trainer.py:231-237): a slot plays WHOLE episodes until it holds
``>= batch_size`` steps -- its last episode overshoots -- and then halts (the lock-step loop runs
``batch_size + max_steps - 1`` iterations when episodes can end early, ``ceil(batch_size /
max_steps) * max_steps`` when they cannot; halted slots leave null records with ``valid = 0``).
``args.batch_boundary = 'cut'`` selects the round-1 behaviour instead (a fixed number of lock-steps,
episodes still open at the end are cut there).

Rollout (the hot path): one lock-step iteration is a handful of kernel launches and no host
synchronisation:
  encoder (index form from the env state, or obs-gather + dense encoder)
  -> policy step (comm mean, C, LSTM, heads, sampling; wgmma tensor-core or fp32 SIMT kernels)
  -> env step + Trainer.get_episode bookkeeping + auto-reset (ic3_rollout_io).
Dense observations on the tensor-core path (``_overlap_obs``): the policy step takes x from the env state, and a side
stream writes the [B, N, O] observation block of the same state concurrently (ic3_*_obs_bounded); the env step waits
for that write.
The whole T-step sequence can be captured once into a CUDA graph (``use_graph``).

Gradient (``compute_grad``, trainer.py:128-225; scope row 8(f)-1): with ``record_for_grad`` the env step kernels record
the inputs of every policy step and the env state its observation is taken from (predator-prey: positions; traffic
junction: positions, alive, last action, route), the same records for every ``grad_impl``; an observation is rebuilt
from them when the backward needs it (``_record_state``).  Returns by a CUDA scan kernel,
then the policy forward is RECOMPUTED with differentiable torch ops (fp32, batched over all slots)
in windows of ``grad_window`` steps processed last-to-first; (h, c) at every window start are
checkpointed during the rollout and the gradient w.r.t. them is handed to the previous window,
so back-propagation through time is exact (truncated only where the reference truncates it:
``detach_gap``, trainer.py:56-60, and episode starts).

With the hand-written BPTT kernels (``grad_impl = 'kernels'``, the default where supported) the backward needs every
step's (h, c).  ``record_mode == 'full'``: the policy step writes them into ``rec_h / rec_c [T+1, B*N, H]``, 2 (T+1) B N H
4 bytes (48.7 GB at predator-prey hard, 8192 slots, batch 500).  When those do not fit in the device memory left after
the other buffers (``RECORD_BYTES_LIMIT``, ``RECORD_MARGIN_BYTES``), ``record_mode == 'window'``: the rollout keeps (h, c)
only at every ``grad_window``-th step plus max |c| per step, and the backward re-runs the tensor-core policy step over
one window at a time from its checkpoint into one of two window buffers, just ahead of the BPTT kernels of that window
(``_recompute_window``).  The recompute is bit-exact, so the gradient equals the full records' bit for bit.
The tanh RNN (models.RNN with rnn_type 'MLP', the IC / IRIC baselines, on the SIMT policy kernel) has no c: its records
are h alone, (T+1) B N H 4 bytes (24.3 GB at predator-prey hard, 8192 slots, batch 500), and its windows are re-run with
the index encoder and the SIMT step.

The non-recurrent tanh policies (models.MLP, CommNet / IC3Net without --recurrent) carry nothing from one step to the
next.  With ``grad_impl = 'kernels_ff'`` their gradient comes from the kernels of ic3_ff_grad_* (csrc/bptt_tc.cu): no
hidden-state record or checkpoint at all; the backward re-runs the forward from the env-state records over chunks of K
consecutive lock-steps (K*B env slots at once, K from the memory the device has left, ``FF_CHUNK_STEPS``), with the
products of the backward on the tensor cores (csrc/ff_grad_tc.cu).

Update (``train_batch`` -> ``update``, trainer.py:245-256): gradient zeroing, rollout, gradient, statistics vector,
RMSprop with the step count read on the device and the weight re-pack, with one host read at the end, which raises on a
device error flag of the rollout or the gradient (the step is then skipped).  ``graph_update`` replays the same phases
from CUDA graphs instead of running them; MultiGPUTrainer runs its all-reduces between them.
"""
import argparse
import ctypes as C
import math
from collections import namedtuple

import torch
import torch.nn.functional as F

from . import _lib, data, eval_trace
from .models import Random
from .optim import FlatRMSprop
from .utils import merge_stat

Transition = namedtuple('Transition', ('state', 'action', 'action_out', 'value', 'episode_mask',
                                       'episode_mini_mask', 'next_state', 'reward', 'misc'))

RolloutBatch = namedtuple('RolloutBatch', ('action', 'logp', 'value', 'reward', 'episode_mask',
                                           'episode_mini_mask', 'alive_mask', 'valid'))

# The env state a policy step's observation is taken from, recorded for compute_grad: record buffer [T, ...] ->
# (env attribute holding the live state, ic3_*_state field, ic3_rollout_io field through which the env step records it)
PP_RECORDS = (('s_loc', 'loc', 'loc', 'snap_pp_loc'),)
TJ_RECORDS = (('s_tjloc', 'car_loc', 'loc', 'snap_tj_loc'), ('s_tjalive', 'alive_mask', 'alive', 'snap_tj_alive'),
              ('s_tjlast', 'car_last_act', 'last_act', 'snap_tj_last_act'),
              ('s_tjroute', 'route_id', 'route_id', 'snap_tj_route_id'))

# What a lock-step writes in every slot's buffers (models.Random has no h or c): the state a warm-up pass before a CUDA
# graph capture rewinds (_capture)
SLOT_STATE = ('fresh', 'comm', 'alive', 't_ep', 'h', 'c', 'halted', 'stat_reward', 'stat_comm', 'stat_success',
              'stat_episodes', 'stat_steps', 'err')


def policy_forward_torch(net, x, h, c, g, n_alive):
    """Differentiable torch restatement of the policy step the kernels run (comm.py:134-244 for every variant of
    ic3_policy_cfg.cell / passes / x_tanh / h_from_x), on the module's own parameters.  x: encoder output [R, H];
    h, c: [R, H] entering the step; g: comm gate per agent [B, N] (alive * comm_action); n_alive: [B, 1].
    Returns (h', c', value [R, 1], [log-probs per head [R, na]])."""
    w, cp = net._kernel_weights(), net._cfg_proto
    B, N = g.shape
    H = x.shape[1]
    lstm = cp['cell'] == _lib.CELL_LSTM
    if cp['x_tanh']:
        x = torch.tanh(x)                                                              # comm.py:127-128
    hid = x if cp['h_from_x'] else h                                                   # comm.py:129
    den = torch.where(n_alive > 1, n_alive - 1, torch.ones_like(n_alive)) if cp['comm_avg'] else torch.ones_like(n_alive)
    gg = g.unsqueeze(-1)
    for ps in range(max(1, cp['passes'])):                                             # comm.py:179
        if cp['comm_mask_zero'] or N < 2:
            S = torch.zeros_like(hid)
        else:
            hv = hid.view(B, N, H)
            tot = (gg * hv).sum(1, keepdim=True)
            S = (gg * (tot - gg * hv) / den.unsqueeze(-1)).reshape(B * N, H)           # comm.py:181-205
        cvec = F.linear(S, w['c_w'][ps], w['c_b'][ps])                                 # comm.py:206
        if lstm:
            gates = F.linear(x + cvec, w['w_ih'], w['b_ih']) + F.linear(hid, w['w_hh'], w['b_hh'])   # comm.py:211-218
            gi, gf, gq, go = gates.chunk(4, dim=1)
            c = torch.sigmoid(gf) * c + torch.sigmoid(gi) * torch.tanh(gq)
            hid = torch.sigmoid(go) * torch.tanh(c)
        else:
            hid = torch.tanh(x + F.linear(hid, w['f_w'][ps], w['f_b'][ps]) + cvec)     # comm.py:220-224
    value = F.linear(hid, w['value_w'], w['value_b'])                                  # comm.py:228
    logps = [F.log_softmax(F.linear(hid, hw, hb), dim=-1) for hw, hb in zip(w['head_w'], w['head_b'])]
    return hid, c, value, logps


class Trainer(object):
    def __init__(self, args, policy_net, env):
        # models.Random (models.py:37-56): one ic3_random_policy_step per lock-step, no gradient (_enqueue_random)
        self.random_policy = isinstance(policy_net, Random)
        if self.random_policy and args.recurrent:
            raise ValueError("models.Random is not recurrent: --random takes no --recurrent (the reference's "
                             "Random.forward would receive [state, prev_hid] and fail on it)")
        if not self.random_policy and not hasattr(policy_net, 'packed'):
            raise NotImplementedError("Trainer drives policies that run on the CUDA kernels (CommNetMLP, models.MLP, "
                                      "models.RNN, models.Random)")
        self.args = args
        self.policy_net = policy_net
        self.env = env                       # GymWrapper
        self.display = False
        self.last_step = False
        # trainer.py:21-22 RMSprop(lr, alpha=0.97, eps=1e-6) as one kernel over flat buffers (optim.py)
        self.optimizer = FlatRMSprop(policy_net.parameters(), lr=args.lrate, alpha=0.97, eps=1e-6)
        self.params = [p for p in self.policy_net.parameters()]
        self.obs_mode = getattr(args, 'obs_mode', 'index')      # 'index' | 'dense'
        self.use_graph = bool(getattr(args, 'use_graph', False))
        self.is_tj = args.env_name == 'traffic_junction'
        self._records = TJ_RECORDS if self.is_tj else PP_RECORDS
        self.hard = bool(args.hard_attn) and bool(args.commnet)      # hard attention gates (trainer.py:70)
        self.record_for_grad = bool(getattr(args, 'record_for_grad', False))
        self.grad_window = int(getattr(args, 'grad_window', 40))
        # compute_grad implementation: 'kernels' = hand-written BPTT (csrc/bptt_tc.cu; tensor-core policy path with the
        # LSTM cell and 1..4 comm passes, or the tanh RNN without communication on the SIMT path; at most 7 action
        # logits, observation pattern of <= 512 columns), 'kernels_ff' = the non-recurrent tanh policies' kernels,
        # 'autograd' = windowed recompute under torch autograd.  Default: kernels when the configuration allows.
        self.grad_impl = getattr(args, 'grad_impl', None) or 'auto'
        if self.grad_impl not in ('auto', 'kernels', 'kernels_ff', 'autograd'):
            raise ValueError("grad_impl must be 'auto', 'kernels', 'kernels_ff' or 'autograd', not %r" % (self.grad_impl,))
        self.grad_kernels = False
        self.grad_ff = False
        self._bptt = None
        self._buf = None
        self._record_mode = None             # 'full' | 'window' per allocation (record_mode)
        self._ff_K = None                    # graph_update: kernels_ff chunk length frozen into the captured update
        self.ff_chunk_pin = None             # kernels_ff chunk length of a resumed run's last update (load_rank_state)
        self._graphs = {}                    # 'rollout' | 'evaluate' | 'update' -> (key, graphs, result) (_replay)
        self._side = None                    # stream of the dense observation writer (_overlap_obs)
        # graph_update: train_batch replays the whole update from CUDA graphs (update)
        self.graph_update = bool(getattr(args, 'graph_update', False))
        self.update_captures = 0             # graph_update: how often the update was captured
        if self.random_policy and self.graph_update:
            raise NotImplementedError("graph_update replays a gradient update; models.Random has neither gradient nor "
                                      "optimizer step, and its rollout is replayed by use_graph")
        if self.random_policy:
            # nothing to record for a gradient: compute_grad reaches no parameter (trainer.py:223), so .grad stays None
            self.record_for_grad = False
            for p in self.params:
                p.grad = None
            return
        # encoder layout of this environment (class terms / counts summed separately, comm.py set_obs_layout); the
        # fused index encoder's per-position table of the class terms belongs to the policy (encoder_table)
        policy_net.set_obs_layout(*getattr(env.env, 'obs_layout', (0, 0, 0)))
        if self.record_for_grad and self.grad_impl in ('auto', 'kernels'):
            # the library decides which configurations its kernels cover; an LSTM cell also needs the tensor-core path,
            # whose weight image and policy step the kernels re-use
            cfg = policy_net.policy_cfg(env.env.nenvs)
            ok = ((cfg.cell == _lib.CELL_TANH or policy_net.policy_impl == 'tc') and
                  self._bptt_workspace_bytes(cfg) > 0)
            if self.grad_impl == 'kernels' and not ok:
                raise NotImplementedError("grad_impl='kernels' needs the tensor-core policy path (hid_size 128, LSTM "
                                          "cell) with the per-position encoder table, or the tanh RNN without "
                                          "communication at hid_size 128; <= 7 action logits and a small vision "
                                          "window")
            self.grad_kernels = ok
        if self.grad_impl == 'auto':
            self.grad_impl = 'kernels' if self.grad_kernels else 'autograd'
        if self.graph_update and self.record_for_grad and self.grad_impl == 'autograd':
            raise NotImplementedError("graph_update needs the gradient kernels (grad_impl 'kernels' or 'kernels_ff'): "
                                      "the torch recompute of grad_impl='autograd' cannot be captured into a CUDA graph")
        if self.graph_update and getattr(policy_net, 'forward_grad', None) == 'kernels':
            raise NotImplementedError("graph_update does not cover forward_grad='kernels': that policy's forward is "
                                      "differentiated by torch autograd, which cannot be captured into a CUDA graph")
        # the non-recurrent tanh policies' kernels (ic3_ff_grad_*): no (h, c) records or checkpoints
        self.grad_ff = self.record_for_grad and self.grad_impl == 'kernels_ff'
        if self.grad_ff:
            e = env.env
            cfg = policy_net.policy_cfg(e.nenvs)
            if int(_lib.load().ic3_ff_grad_workspace_bytes(C.byref(self._ff_plan(cfg, None, e.nenvs * args.nagents)))) == 0:
                raise NotImplementedError("grad_impl=%r covers the non-recurrent tanh policies (models.MLP, "
                                          "CommNet / IC3Net without --recurrent, 1..%d comm passes) at hid_size 128 with "
                                          "<= 7 action logits, a vision window of <= 5 x 5 cells and an observation "
                                          "pattern of <= 512 columns" % (self.grad_impl, _lib.MAX_PASSES))

    def _policy_cfg(self, e=None):
        """ic3_policy_cfg of the policy step over this GPU's slots of env e (default: the training env), with the env's
        Philox key and env ids."""
        e = self.env.env if e is None else e
        cfg = self.policy_net.policy_cfg(e.nenvs)
        cfg.seed, cfg.env_id0 = e.cfg.seed, e.cfg.env_id0
        return cfg

    def _bptt_plan(self, cfg, w=None, x_table=None):
        e, args = self.env.env, self.args
        return _lib.BpttPlan(cfg=C.pointer(cfg), w=None if w is None else C.pointer(w),
                             pp_env=None if self.is_tj else C.pointer(e.cfg), tj_env=C.pointer(e.cfg) if self.is_tj else None,
                             x_table=x_table, value_coeff=float(args.value_coeff), entr=float(args.entr), workspace=None)

    def _bptt_workspace_bytes(self, cfg):
        """ic3_bptt_workspace_bytes of the policy configuration cfg on this environment (0: not covered)."""
        return int(_lib.load().ic3_bptt_workspace_bytes(C.byref(self._bptt_plan(cfg))))

    def _encoder_table(self, cfg=None, w=None, e=None):
        """The policy's per-position encoder table for env e (default: the training env; CommNetMLP.encoder_table),
        built from its current packed weights; cfg and w are accepted for callers that hold them and are not needed."""
        return self.policy_net.encoder_table(self.env.env if e is None else e)

    # ------------------------------------------------------------------ buffers
    def _slot_buffers(self, B, T, dev):
        """What every run of the lock-step loop over B slots needs: episode state, statistics, T steps of action /
        log-prob / value and, for a policy with weights, h, c and x."""
        N, H = self.args.nagents, self.args.hid_size
        nh = len(self.args.naction_heads)
        A = sum(self.args.naction_heads)
        z = lambda *s, dtype=torch.float32: torch.zeros(*s, dtype=dtype, device=dev)
        b = dict(T=T, comm=z(B, N, dtype=torch.uint8), alive=torch.ones(B, N, dtype=torch.uint8, device=dev),
                 fresh=torch.ones(B, dtype=torch.uint8, device=dev), t_ep=z(B, dtype=torch.int32),
                 action=z(T, B, N, nh, dtype=torch.int32), logp=z(T, B, N, A), value=z(T, B * N), step_reward=z(B, N),
                 stat_reward=z(B, N), stat_comm=z(B, N), stat_success=z(B, dtype=torch.int32),
                 stat_episodes=z(B, dtype=torch.int32), stat_steps=z(B, dtype=torch.int32),
                 err=z(1, dtype=torch.int32), halted=z(B, dtype=torch.uint8), statvec=z(4 + 2 * N, dtype=torch.float64))
        if not self.random_policy:            # models.Random has no encoder or recurrent state
            b.update(h=z(B * N, H), c=z(B * N, H), x=z(B * N, H))
        return b

    def _alloc(self, T):
        # the previous buffers, and the graphs that run on them, go back to the allocator before the records are sized
        self._buf = None
        for name in ('rollout', 'update'):
            self._graphs.pop(name, None)
        e = self.env.env
        B, N, H = e.nenvs, self.args.nagents, self.args.hid_size
        dev = e.device
        A = sum(self.args.naction_heads)
        z = lambda *s, dtype=torch.float32: torch.zeros(*s, dtype=dtype, device=dev)
        b = self._slot_buffers(B, T, dev)
        b.update(reward=z(T, B, N), emask=z(T, B, dtype=torch.uint8), mini=z(T, B, N, dtype=torch.uint8),
                 ralive=z(T, B, N, dtype=torch.uint8), valid=z(T, B, dtype=torch.uint8))
        if self.random_policy:                # no observation or recurrent state
            self._buf = b
            return b
        if self.obs_mode == 'dense':
            b['obs'] = torch.empty(B, N, self.env.observation_dim, dtype=torch.float32, device=dev)
        if self.record_for_grad:
            # the inputs of every policy step and the env state its observation is taken from (_record_state), then
            # (h, c) in one of three forms:
            #   torch paths  (h, c) checkpoints at the starts of grad_window-step windows (_forward_window re-runs them)
            #   BPTT kernels (_record_bytes):
            #     'full'   rec_h, rec_c [T+1, B*N, H] -- the policy step writes them straight into the record,
            #              rec_h[t] -> rec_h[t + 1];
            #     'window' the checkpoints plus max |c| of every step; the backward re-runs the policy step over one
            #              window at a time (_recompute_window)
            b.update(s_fresh=z(T, B, dtype=torch.uint8), s_comm=z(T, B, N, dtype=torch.uint8),
                     s_alive=z(T, B, N, dtype=torch.uint8), s_tep=z(T, B, dtype=torch.int32))
            for key, attr, _, _ in self._records:
                live = getattr(e, attr)
                b[key] = z(T, *live.shape, dtype=live.dtype)
            W = self.grad_window
            nw = (T + W - 1) // W
            self._record_mode = self._pick_record_mode(T) if self.grad_kernels else None
            hc = not self._h_only_records()          # the tanh RNN's kernels keep h alone: it has no c
            if self._record_mode == 'full':
                b['rec_h'] = torch.empty(T + 1, B * N, H, device=dev)
                if hc:
                    b['rec_c'] = torch.empty(T + 1, B * N, H, device=dev)
            elif not self.grad_ff:          # kernels_ff re-runs every step from the env-state records alone
                b['ck_h'] = z(nw, B * N, H)
                if hc:
                    b['ck_c'] = z(nw, B * N, H)
            if self._record_mode == 'window':
                nb, L = min(nw, self._window_buffers()), min(W, T)      # window k lives in buffer k % _window_buffers()
                e_ = lambda *s: torch.empty(*s, device=dev)
                b.update(win_h=[e_(L, B * N, H) for _ in range(nb)], win_value=e_(B * N), win_logp=e_(B * N, A))
                if hc:
                    b.update(c_abs=z(T), win_c=[e_(L, B * N, H) for _ in range(nb)])
        self._buf = b
        return b

    # The BPTT kernels' (h, c) records.  What the device has for them is measured when the rollout buffers have been
    # allocated: free memory plus the caching allocator's unused reserve, minus RECORD_MARGIN_BYTES and the compute_grad
    # temporaries (RECORD_TEMP_FACTOR float32 [T, B, N] tensors: returns, advantages and their intermediates).  Full
    # records are kept while they take at most RECORD_BYTES_LIMIT bytes (None: what the device has); beyond that the
    # records switch to windows of grad_window steps, which must fit in what the device has.
    RECORD_BYTES_LIMIT = None
    RECORD_MARGIN_BYTES = 2 << 30            # one-pass BPTT workspace (~0.9 GB at 81 920 rows) and allocator slack;
    #                                          what comm_passes > 1 adds to the workspace is counted on top (_pick_record_mode)
    RECORD_TEMP_FACTOR = 6

    @property
    def record_mode(self):
        """How the BPTT kernels get every step's (h, c): 'full' records or 'window' recompute (None without the BPTT
        kernels).  Chosen per rollout length when the buffers are allocated; before the first rollout, the choice
        run_batch would make now."""
        if not (self.record_for_grad and self.grad_kernels):
            return None
        if self._buf is None:
            return self._pick_record_mode(self.batch_plan()[0])
        return self._record_mode

    def _window_buffers(self):
        # windows are re-run two ahead of the backward (_compute_grad_kernels); one-step windows need a third buffer
        return 2 if self.grad_window >= 2 else 3

    def _h_only_records(self):
        """The BPTT kernels of the tanh RNN record h alone (no c, no max |c|)."""
        return self.grad_kernels and self.policy_net._cfg_proto['cell'] == _lib.CELL_TANH

    def _record_bytes(self, T):
        """{'full': bytes of rec_h + rec_c, 'window': bytes of the checkpoints + window buffers} for T steps (h alone
        for the tanh RNN)."""
        R, H, W = self.env.env.nenvs * self.args.nagents, self.args.hid_size, self.grad_window
        row = R * H * 4
        nw = (T + W - 1) // W
        nb = min(nw, self._window_buffers())
        if self._h_only_records():
            return dict(full=(T + 1) * row, window=nw * row + nb * min(W, T) * row)
        return dict(full=2 * (T + 1) * row, window=2 * nw * row + 2 * nb * min(W, T) * row + T * 4)

    def _bptt_extra_bytes(self):
        """Bytes the BPTT workspace of this policy needs beyond the one-pass workspace RECORD_MARGIN_BYTES covers: the
        per-pass states, weight images and partials of comm_passes > 1 (0 with one pass)."""
        if int(self.args.comm_passes) <= 1:
            return 0
        cfg = self.policy_net.policy_cfg(self.env.env.nenvs)
        one = self.policy_net.policy_cfg(self.env.env.nenvs)
        one.passes = 1
        return max(0, self._bptt_workspace_bytes(cfg) - self._bptt_workspace_bytes(one))

    def _device_bytes_free(self):
        """The device's free memory plus the caching allocator's unused reserve."""
        dev = self.env.env.device
        free, _ = torch.cuda.mem_get_info(dev)
        return free + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)

    def _pick_record_mode(self, T):
        need = self._record_bytes(T)
        avail = (self._device_bytes_free() - self.RECORD_MARGIN_BYTES - self._bptt_extra_bytes()
                 - self.RECORD_TEMP_FACTOR * T * self.env.env.nenvs * self.args.nagents * 4)
        limit = avail if self.RECORD_BYTES_LIMIT is None else min(avail, self.RECORD_BYTES_LIMIT)
        if need['full'] <= limit:
            return 'full'
        if need['window'] <= avail:
            return 'window'
        raise RuntimeError("the BPTT kernels need %.3g GB for the (h, c) records of %d steps in windows of %d steps "
                           "(%.3g GB as full records) but the device has %.3g GB for them; reduce --nenvs or "
                           "--batch_size" % (need['window'] / 1e9, T, self.grad_window, need['full'] / 1e9,
                                             max(avail, 0) / 1e9))

    # ------------------------------------------------------------------ rollout
    def _fused_x(self):
        """Index-form observations on the tensor-core policy path: the encoder runs inside the policy step."""
        return self.obs_mode != 'dense' and self.policy_net.fuses_encoder(self.env.env)

    # Smaller observation blocks per step keep the fused gather + encoder: their write is short and latency-bound in the
    # persistent writer (measured on an H100: predator-prey easy, 2.9 MB, 3 % slower with the overlap; traffic-junction
    # medium, 20 MB, 1 % faster; predator-prey hard, 1.19 GB, 9 % faster).
    OVERLAP_MIN_OBS_BYTES = 8 << 20

    def _overlap_obs(self, e=None):
        """Dense observations on the tensor-core policy path: the policy step computes x from the env state (the fused
        index encoder; without the per-position table, which measured no faster beside the writer, so dense mode never
        builds it) and the observation block is written concurrently on a side stream.  Not for blocks smaller than
        OVERLAP_MIN_OBS_BYTES."""
        if self.obs_mode != 'dense':
            return False
        e = self.env.env if e is None else e
        if e.nenvs * self.args.nagents * self.env.observation_dim * 4 < self.OVERLAP_MIN_OBS_BYTES:
            return False
        return self.policy_net.fuses_encoder(e)

    def _enqueue(self, T, quota=0, b=None, e=None, episodes=0, greedy=False, recorder=None):
        """Enqueue T lock-step iterations on the current stream (no host sync).  quota > 0: reference batch
        boundary -- a slot halts at the first episode end with >= quota steps (ic3_rollout_io.batch_size);
        quota = 0: episodes still open at iteration T-1 are cut there.  b, e: buffers and env (default: the training
        rollout's; evaluate passes its own, which hold no records and one lock-step of action / log-prob / value
        scratch, and no observation block: x comes from the env state); episodes > 0: episode quota
        (ic3_rollout_io.episodes); greedy: argmax actions (ic3_policy_cfg.greedy); recorder: an eval_trace.Recorder
        that keeps every lock-step before its policy step and between its policy step and its env step
        (evaluate_trace)."""
        b = self._buf if b is None else b
        e = self.env.env if e is None else e
        if self.random_policy:
            return self._enqueue_random(T, quota, b, e, episodes, recorder)
        net = self.policy_net
        lib = _lib.load()
        B = e.nenvs
        cfg = self._policy_cfg(e)
        cfg.greedy = int(greedy)
        w = net.packed()
        s = _lib.stream()
        ws, _ = net.workspace(B)          # tensor-core path scratch (None for the fp32 SIMT kernel)
        rec = self.record_for_grad and 's_fresh' in b
        full = rec and self._record_mode == 'full'    # the policy step writes (h, c) straight into the records
        window = rec and self._record_mode == 'window'    # (h, c) checkpoints + max |c| per step (_alloc)
        hc = not self._h_only_records()               # the tanh RNN's kernel records: h alone
        dense = 'obs' in b                            # _alloc makes the block for obs_mode 'dense'
        # dense observations written on a side stream while the policy step runs (see _overlap_obs)
        overlap = dense and self._overlap_obs(e)
        # tensor-core path: the index encoder is fused into the policy step (x never leaves the operand image)
        fused_x = (not dense and net.fuses_encoder(e)) or overlap
        src = {}
        if fused_x:
            src = dict(_lib.env_source(e.cfg, e.state),
                       x_table=None if overlap else _lib.ptr(self._encoder_table(e=e)))
        if overlap:
            main = torch.cuda.current_stream()
            if self._side is None or self._side.device != main.device:
                self._side = torch.cuda.Stream(device=main.device)
            side = self._side
            obs_write = lib.ic3_tj_obs_bounded if self.is_tj else lib.ic3_pp_obs_bounded
        snap = {}
        if rec:
            snap = dict(snap_T=T, snap_fresh=b['s_fresh'].data_ptr(), snap_comm=b['s_comm'].data_ptr(),
                        snap_alive=b['s_alive'].data_ptr(), snap_tep=b['s_tep'].data_ptr(),
                        **{field: b[key].data_ptr() for key, _, _, field in self._records})
        for t in range(T):
            if rec:
                if t == 0:          # inputs of the first step; the env step kernels record those of every later step
                    b['s_fresh'][0].copy_(b['fresh'])
                    b['s_comm'][0].copy_(b['comm'])
                    b['s_alive'][0].copy_(b['alive'])
                    b['s_tep'][0].copy_(b['t_ep'])
                    for key, attr, _, _ in self._records:
                        b[key][0].copy_(getattr(e, attr))
                if not full and not self.grad_ff and t % self.grad_window == 0:
                    b['ck_h'][t // self.grad_window].copy_(b['h'])
                    if hc:
                        b['ck_c'][t // self.grad_window].copy_(b['c'])
            if overlap:
                # the writer reads the state the previous env step left and must finish before this step's env step
                # moves the agents (the join below)
                side.wait_stream(main)
                _lib.check(obs_write(C.byref(e.cfg), C.byref(e.state), b['obs'].data_ptr(), side.cuda_stream))
            elif dense:
                # gather + encode in one kernel: the observation block is written in full and x is summed from the
                # same per-cell records, so the block is never read back
                obs_enc = lib.ic3_tj_obs_encode if self.is_tj else lib.ic3_pp_obs_encode
                _lib.check(obs_enc(C.byref(e.cfg), C.byref(e.state), C.byref(cfg), C.byref(w), b['obs'].data_ptr(),
                                   b['x'].data_ptr(), s))
            elif fused_x:
                pass
            elif self.is_tj:
                _lib.check(lib.ic3_tj_encoder_index(C.byref(e.cfg), C.byref(e.state), C.byref(cfg), C.byref(w),
                                                    b['x'].data_ptr(), s))
            else:
                _lib.check(lib.ic3_pp_encoder_index(C.byref(e.cfg), C.byref(e.state), C.byref(cfg), C.byref(w),
                                                    b['x'].data_ptr(), s))
            hin, hout = (b['rec_h'][t], b['rec_h'][t + 1]) if full else (b['h'], b['h'])
            cin, cout = (b['rec_c'][t], b['rec_c'][t + 1]) if full and hc else (b['c'], b['c'])
            r = t % b['T']                    # record row: t, or 0 in evaluate's one-step scratch
            io = _lib.PolicyIO(x=None if fused_x else b['x'].data_ptr(), h=hin.data_ptr(), c=cin.data_ptr(),
                               comm_action=b['comm'].data_ptr() if self.hard else None, alive=b['alive'].data_ptr(),
                               fresh=b['fresh'].data_ptr(), tick=e.tick.data_ptr(), draws=None,
                               h_out=hout.data_ptr(), c_out=cout.data_ptr(), value=b['value'][r].data_ptr(),
                               logp=b['logp'][r].data_ptr(), action=b['action'][r].data_ptr(),
                               workspace=_lib.ptr(ws), err=b['err'].data_ptr(), **src)
            if recorder is not None:
                recorder.pre_step(t, s)
            _lib.check(lib.ic3_policy_step(C.byref(cfg), C.byref(w), C.byref(io), s))
            if window and hc:
                # max |c'| of this step: the backward's operand scale needs the bound over every step's c before it
                # re-runs any window, the same value a full record gives (_compute_grad_kernels)
                torch.linalg.vector_norm(b['c'], math.inf, out=b['c_abs'][t])
            if overlap:
                main.wait_stream(side)
            if recorder is not None:
                recorder.step(t, s)
            self._env_step(t, T, quota, snap, s, b, e, episodes, recorder)
        if recorder is not None:
            recorder.finish(T, s)

    def _env_step(self, t, T, quota, snap, s, b=None, e=None, episodes=0, recorder=None):
        """Env step of lock-step iteration t on the actions the policy step wrote to the records, with the
        Trainer.get_episode bookkeeping and auto-reset (ic3_rollout_io; ``snap``: its snap_* fields).  b, e, episodes,
        recorder: see _enqueue; a record evaluate's buffers do not hold is passed as NULL."""
        b = self._buf if b is None else b
        e = self.env.env if e is None else e
        args = self.args
        lib = _lib.load()
        nh = len(args.naction_heads)
        act = b['action'][t % b['T']]
        rec = lambda k: _lib.ptr(b.get(k))
        r = _lib.RolloutIO(t=t, max_steps=args.max_steps, nheads=nh, hard_attn=int(self.hard),
                           comm_action_one=int(bool(args.comm_action_one)),
                           last=int(t == T - 1 and quota <= 0 and episodes <= 0), batch_size=int(quota),
                           episodes=int(episodes), halted=b['halted'].data_ptr(), rec_valid=rec('valid'), **snap,
                           action=act.data_ptr(), t_ep=b['t_ep'].data_ptr(),
                           fresh=b['fresh'].data_ptr(), comm_next=b['comm'].data_ptr(),
                           alive_next=b['alive'].data_ptr(), rec_reward=rec('reward'),
                           rec_episode_mask=rec('emask'), rec_mini_mask=rec('mini'),
                           rec_alive=rec('ralive'), stat_reward=b['stat_reward'].data_ptr(),
                           stat_comm=b['stat_comm'].data_ptr(), stat_success=b['stat_success'].data_ptr(),
                           stat_episodes=b['stat_episodes'].data_ptr(), stat_steps=b['stat_steps'].data_ptr(),
                           **(recorder.rollout_fields() if recorder is not None else {}))
        if self.is_tj:
            _lib.check(lib.ic3_tj_step(C.byref(e.cfg), C.byref(e.state), act.data_ptr(), nh, None,
                                       b['step_reward'].data_ptr(), None, b['err'].data_ptr(), C.byref(r), s))
        else:
            _lib.check(lib.ic3_pp_step(C.byref(e.cfg), C.byref(e.state), act.data_ptr(), nh,
                                       b['step_reward'].data_ptr(), None, b['err'].data_ptr(), C.byref(r), s))

    def random_cfg(self, e=None):
        """ic3_policy_cfg of the Random policy step: the fields ic3_random_policy_step reads (B, N, heads, Philox key
        and env ids of this GPU's slots of env e, default the training env)."""
        e, heads = self.env.env if e is None else e, list(self.args.naction_heads)
        return _lib.PolicyCfg(B=e.nenvs, N=self.args.nagents, nheads=len(heads),
                              head_dim=(C.c_int32 * _lib.MAX_HEADS)(*heads), env_id0=e.cfg.env_id0, seed=e.cfg.seed)

    def _enqueue_random(self, T, quota, b, e, episodes=0, recorder=None):
        """_enqueue for models.Random: per lock-step iteration one ic3_random_policy_step (value, log-probs and actions
        into the records, from the env's action tick) and the env step."""
        lib = _lib.load()
        cfg = self.random_cfg(e)
        s = _lib.stream()
        for t in range(T):
            r = t % b['T']
            io = _lib.PolicyIO(tick=e.tick.data_ptr(), value=b['value'][r].data_ptr(), logp=b['logp'][r].data_ptr(),
                               action=b['action'][r].data_ptr())
            _lib.check(lib.ic3_random_policy_step(C.byref(cfg), C.byref(io), None, s))
            if recorder is not None:
                recorder.step(t, s)
            self._env_step(t, T, quota, {}, s, b, e, episodes, recorder)
        if recorder is not None:
            recorder.finish(T, s)

    def _episode_boundary(self, epoch, b=None, e=None):
        b = self._buf if b is None else b
        e = self.env.env if e is None else e
        if self.is_tj:
            e.reset(epoch, want_obs=False)
        else:
            e.reset(want_obs=False)
        for k in ('stat_reward', 'stat_comm', 'stat_success', 'stat_episodes', 'stat_steps', 't_ep', 'halted'):
            b[k].zero_()
        b['fresh'].fill_(1)

    def _begin(self, T, epoch, b=None, e=None):
        """Start a run of T lock-step iterations on buffers b and env e (default: the training rollout's, allocated
        anew when T changes): fresh episodes in every slot (trainer.py:28-32, 45-51; the TJ curriculum may move
        cfg.spawn_thr), the error word zeroed, and the packed weights and e's encoder table brought up to date outside
        any graph capture (_refresh_weights).  Returns (b, e)."""
        if b is None:
            if self._buf is None or self._buf['T'] != T:
                self._alloc(T)
            b = self._buf
        e = self.env.env if e is None else e
        self._episode_boundary(epoch, b, e)
        b['err'].zero_()
        self._refresh_weights(b, e)
        return b, e

    def _refresh_weights(self, b, e, force=False):
        """Re-pack the weights and re-build the encoder table a run on buffers b and env e reads (none with a dense
        observation block) if the parameters changed since they were built; with force always."""
        if not self.random_policy:
            self.policy_net.packed(force=force)
            if 'obs' not in b:
                self.policy_net.encoder_table(e, force=force)

    def rollout(self, T, epoch=0, quota=0):
        """T lock-step iterations from fresh episodes in every slot (``quota``: see _enqueue).  Returns a
        RolloutBatch of stacked [T, B, ...] device tensors (views of the trainer's record buffers)."""
        b, e = self._begin(T, epoch)
        self._run_rollout(T, quota, b, e)
        return RolloutBatch(action=b['action'], logp=b['logp'], value=b['value'].view(T, e.nenvs, -1),
                            reward=b['reward'], episode_mask=b['emask'], episode_mini_mask=b['mini'],
                            alive_mask=b['ralive'], valid=b['valid'])

    def _run_rollout(self, T, quota, b, e):
        """Enqueue the training rollout on buffers b and env e, replayed from the 'rollout' CUDA graph with use_graph."""
        run = lambda: self._enqueue(T, quota)
        if self.use_graph:
            self._replay('rollout', self._graph_key(T, e, int(quota)), b, e, [run])
        else:
            run()

    def _graph_key(self, T, e, *extras):
        """Key of a run of T lock-steps on env e captured into CUDA graphs: kernel arguments passed BY VALUE are frozen
        into a graph, so everything of that kind that can change between runs is part of the key (the TJ curriculum
        moves cfg.spawn_thr, traffic_junction_env.py:196-200,620-626; a re-seeded env changes cfg.seed), with the
        caller's own such values in extras."""
        return (T, int(getattr(e.cfg, 'spawn_thr', 0)), int(e.cfg.seed), int(e.cfg.env_id0), e.nenvs) + extras

    def _replay(self, name, key, b, e, phases, between=None, restore=()):
        """Run phases on buffers b and env e by replaying the CUDA graphs cached under name, captured first (_capture)
        when the cache holds none for this key.  Returns (what phases[0] returned, whether they were captured now)."""
        entry = self._graphs.get(name)
        captured = entry is None or entry[0] != key
        if captured:
            entry = self._graphs[name] = (key,) + self._capture(b, e, phases, between, restore)
        _, graphs, out = entry
        graphs[0].replay()
        for g in graphs[1:]:
            between(out)
            g.replay()
        return out, captured

    def _capture(self, b, e, phases, between=None, restore=()):
        """CUDA graphs of phases on buffers b and env e, not yet replayed: phases[0]() returns r (or None), each later
        phase is called with r.  A warm-up pass (lazy library state, allocator, workspaces) runs first and is rewound --
        env state and RNG ticks, b's SLOT_STATE, the tensors in restore -- and the weights are re-packed (the warm-up may
        have packed updated ones, and restored parameters keep their version counters), so the capture starts where an
        eager run would.  One graph holds all phases; with between(r), an eager step between phases (MultiGPUTrainer's
        all-reduces), each phase is a graph of its own in the first one's memory pool.  Returns (graphs, r)."""
        snap = e.snapshot()
        saved = [(t, t.clone()) for t in [b[k] for k in SLOT_STATE if k in b] + list(restore)]
        out = phases[0]()
        for phase in phases[1:]:
            if between is not None:
                between(out)
            phase(out)
        torch.cuda.synchronize()
        e.restore(snap)
        for t, v in saved:
            t.copy_(v)
        self._refresh_weights(b, e, force=True)
        graphs = [torch.cuda.CUDAGraph()]
        with torch.cuda.graph(graphs[0]):
            out = phases[0]()
            if between is None:
                for phase in phases[1:]:
                    phase(out)
        for phase in phases[1:] if between is not None else ():
            graphs.append(torch.cuda.CUDAGraph())
            with torch.cuda.graph(graphs[-1], pool=graphs[0].pool()):
                phase(out)
        return graphs, out

    def stat_vector(self, b=None, e=None):
        """Device float64 vector [num_episodes, num_steps, success, err flags, reward[N], comm_action[N]] of this
        GPU's slots (one kernel, csrc/returns.cu ic3_stat_reduce); no host synchronisation.  b, e: buffers and env
        (default: the training rollout's)."""
        b = self._buf if b is None else b
        e = self.env.env if e is None else e
        _lib.check(_lib.load().ic3_stat_reduce(e.nenvs, self.args.nagents, b['stat_episodes'].data_ptr(),
                                               b['stat_steps'].data_ptr(), b['stat_success'].data_ptr(),
                                               b['err'].data_ptr(), b['stat_reward'].data_ptr(),
                                               b['stat_comm'].data_ptr() if self.hard else None,
                                               b['statvec'].data_ptr(), _lib.stream()))
        return b['statvec']

    def stat_from_vector(self, v, e=None):
        """Host-side stat dict with the reference's keys (trainer.py:73-75,86-88,109-110,124-125,235) from a
        stat_vector() (of this GPU, or summed over ranks) that has been copied to the host; e: the env it was collected
        on (default: the training env)."""
        args, N = self.args, self.args.nagents
        flags = int(v[3])
        if flags:
            raise RuntimeError("device-side error flag %#x during rollout" % flags)
        stat = dict()
        stat['num_episodes'] = int(round(float(v[0])))
        stat['num_steps'] = int(round(float(v[1])))
        stat['steps_taken'] = stat['num_steps']
        nf = int(getattr(args, 'nfriendly', N))                 # trainer.py:73-75,86-88: friendly / enemy split
        enemy = bool(getattr(args, 'enemy_comm', False))
        stat['reward'] = v[4:4 + nf].copy()
        if enemy:
            stat['enemy_reward'] = v[4 + nf:4 + N].copy()
        if args.hard_attn and args.commnet:
            stat['comm_action'] = v[4 + N:4 + N + nf].copy()
            if enemy:
                stat['enemy_comm'] = v[4 + N + nf:4 + 2 * N].copy()
        if not (not self.is_tj and args.mode == 'competitive'):
            stat['success'] = int(round(float(v[2])))
        if self.is_tj:
            # every episode of the batch reports the same env.stat['add_rate'] (traffic_junction_env.py:249-250),
            # merged by + over episodes and workers (trainer.py:124-125, utils.py:15-29)
            stat['add_rate'] = (self.env.env if e is None else e).add_rate * stat['num_episodes']
        return stat

    def collect_stat(self):
        """Stat dict of the last rollout, summed over the env slots of this GPU (ONE device->host copy)."""
        return self.stat_from_vector(self.stat_vector().cpu().numpy())

    # ------------------------------------------------------------------ reference surface
    def get_episode(self, epoch):
        """Exactly one episode per env slot (trainer.py:26-126): max_steps lock-step iterations, a slot whose
        episode ends early halts (``valid`` = 0 afterwards)."""
        batch = self.rollout(self.args.max_steps, epoch, quota=1)
        return batch, self.collect_stat()

    def episodes_end_early(self):
        """Can an episode end before max_steps?  predator_prey 'mixed' mode only (predator_prey_env.py:273-274);
        traffic_junction never sets episode_over (traffic_junction_env.py:219,252)."""
        return (not self.is_tj) and getattr(self.args, 'mode', 'mixed') == 'mixed'

    def batch_plan(self):
        """(lock-step iterations, quota) of one run_batch."""
        bs, ms = int(self.args.batch_size), int(self.args.max_steps)
        full = int(math.ceil(bs / float(ms))) * ms
        if getattr(self.args, 'batch_boundary', 'reference') == 'cut':
            return full, 0
        return (bs + ms - 1 if self.episodes_end_early() else full), bs

    # ------------------------------------------------------------------ evaluation
    def _eval_state(self):
        """The evaluation environment (args.eval_nenvs slots, default nenvs, built once with data.init) and its buffers.
        Its global env ids follow every rank's training ids: training's are id0 + rank * nenvs + [0, nenvs) with id0 the
        job's first training id (this rank's env_id0 - rank * nenvs), evaluation's id0 + world * nenvs +
        rank * eval_nenvs + [0, eval_nenvs), so its Philox streams never meet training's."""
        if getattr(self, '_eval', None) is not None:
            return self._eval
        tr_env, args = self.env.env, self.args
        ne = int(getattr(args, 'eval_nenvs', None) or tr_env.nenvs)
        dist = torch.distributed
        on = dist.is_available() and dist.is_initialized()
        world, rank = (dist.get_world_size(), dist.get_rank()) if on else (1, 0)
        ea = argparse.Namespace(**vars(args))
        ea.nenvs = ne
        ea.env_id0 = int(tr_env.cfg.env_id0) - rank * tr_env.nenvs + world * tr_env.nenvs + rank * ne
        e = data.init(args.env_name, ea).env
        e.cfg.seed = tr_env.cfg.seed
        self._eval = dict(env=e, buf=self._slot_buffers(ne, 1, e.device))
        return self._eval

    def _eval_prepare(self, episodes, greedy, epoch):
        """Argument checks and the evaluation env's add_rate for an evaluation; returns (env, buffers, lock-steps)."""
        episodes = int(episodes)
        if episodes < 1:
            raise ValueError("evaluate plays at least one episode per slot, not %d" % episodes)
        if greedy and self.random_policy:
            raise ValueError("models.Random has no greedy action: its logits do not depend on the observation")
        ev = self._eval_state()
        e, b = ev['env'], ev['buf']
        if self.is_tj:
            if epoch is None:
                e.set_add_rate(self.env.env)
            else:
                e.curriculum_until(int(epoch))
        return e, b, episodes * int(self.args.max_steps)

    def evaluate_vector(self, episodes=1, greedy=False, epoch=None):
        """evaluate without the host read: the device float64 statistics vector (stat_vector's layout) of the episodes,
        and the evaluation env they were played on."""
        e, b, T = self._eval_prepare(episodes, greedy, epoch)
        episodes = int(episodes)
        self._begin(T, None, b, e)
        run = lambda: self._enqueue(T, 0, b, e, episodes, greedy)
        if self.use_graph:
            self._replay('evaluate', self._graph_key(T, e, episodes, bool(greedy)), b, e, [run])
        else:
            run()
        return self.stat_vector(b, e), e

    def evaluate(self, episodes=1, greedy=False, epoch=None):
        """Play exactly ``episodes`` whole episodes in every slot of the evaluation env (see _eval_state), each slot
        from a fresh reset, with sampled actions or, ``greedy``, the argmax of every head.  Returns the collect_stat
        dict of those episodes (raw sums; num_episodes = episodes * eval_nenvs).  Traffic junction: ``epoch`` sets
        add_rate through the env's curriculum as training reaches it at that epoch; None takes the training env's
        current add_rate.  Training state (env, ticks, buffers, records, graphs) is not touched; the policy is only
        read.  Successive calls continue the evaluation env's random streams."""
        vec, e = self.evaluate_vector(episodes, greedy, epoch)
        return self.stat_from_vector(vec.cpu().numpy(), e)

    def _check_messages(self):
        """Raise NotImplementedError unless the policy is the recurrent (LSTM) CommNet / IC3Net with one comm pass,
        whose messages evaluate_trace(messages=True) records."""
        net, args = self.policy_net, self.args
        if self.random_policy:
            raise NotImplementedError("evaluate_trace(messages=True): models.Random does not communicate")
        if bool(getattr(net, 'args', args).comm_mask_zero):
            raise NotImplementedError("evaluate_trace(messages=True): the policy does not communicate (models.MLP, "
                                      "models.RNN or --comm_mask_zero)")
        if not net.recurrent:
            raise NotImplementedError("evaluate_trace(messages=True) records the recurrent CommNet / IC3Net (LSTM "
                                      "cell); the non-recurrent policy is outside its scope")
        if int(args.comm_passes) != 1:
            raise NotImplementedError("evaluate_trace(messages=True) records one comm pass, not comm_passes %d"
                                      % int(args.comm_passes))

    def evaluate_trace_vector(self, episodes=1, greedy=False, epoch=None, slots=8, comm_map=True, messages=False):
        """evaluate_trace without the host read: (device statistics vector, evaluation env, eval_trace.Recorder holding
        the trajectories and the comm map on the device)."""
        if messages:
            self._check_messages()
        e, b, T = self._eval_prepare(episodes, greedy, epoch)
        episodes = int(episodes)
        slots = eval_trace.parse_slots(slots, e.nenvs)
        key = (T, slots, bool(comm_map), bool(messages))
        rec = self._eval.get('trace')
        if rec is None or rec.key != key:
            self._graphs.pop('evaluate_trace', None)       # its graph writes into the recorder it replaces
            self._eval['trace'] = None
            rec = self._eval['trace'] = eval_trace.Recorder(self, e, b, T, slots, bool(comm_map), bool(messages))
            rec.key = key
        self._begin(T, None, b, e)

        def run():
            rec.begin()
            self._enqueue(T, 0, b, e, episodes, greedy, recorder=rec)
        if self.use_graph:
            self._replay('evaluate_trace', self._graph_key(T, e, episodes, bool(greedy)) + key[1:], b, e, [run])
        else:
            run()
        return self.stat_vector(b, e), e, rec

    def evaluate_trace(self, episodes=1, greedy=False, epoch=None, slots=8, comm_map=True, messages=False):
        """evaluate, recording what the agents do: returns (stat, trace, cmap).  stat is what evaluate returns for the
        same call (the same loop, env, buffers and random streams).  trace (eval_trace.EvalTraceResult) holds every
        lock-step of the recorded slots -- ``slots``: the first K evaluation slots, or a sequence of distinct local slot
        numbers -- as [T, K, ...] numpy arrays, T = episodes * max_steps.  cmap (comm_map; else None): integer counts
        over every slot of visits to each cell and each episode step and, with --hard_attn, of gate openings there
        (ic3_comm_map_step).  messages (recurrent CommNet / IC3Net with one comm pass; NotImplementedError otherwise):
        the trace also holds the hidden state each agent sends, its gate and the vector S it receives (msg_h, msg_gate,
        msg_in), and cmap the message map (msg_* keys, eval_trace.Recorder._message_map).  The trace and the map come
        back in one device->host copy."""
        vec, e, rec = self.evaluate_trace_vector(episodes, greedy, epoch, slots, comm_map, messages)
        stat = self.stat_from_vector(vec.cpu().numpy(), e)
        trace, cmap = rec.to_host()
        return stat, trace, cmap

    def steps_per_batch(self):
        return self.batch_plan()[0]

    def run_batch(self, epoch):
        T, quota = self.batch_plan()
        batch = self.rollout(T, epoch, quota=quota)
        self.stats = self.collect_stat()
        return batch, self.stats

    # ------------------------------------------------------------------ gradient (trainer.py:128-225)
    def _record_state(self, t, k0=0, k1=None):
        """(env cfg, env state) of env slots [k0, k1) as the records hold them entering step t: the live state view with
        the recorded fields substituted (predator-prey: loc; traffic junction: loc, alive, last_act, route_id), which
        are all the encoders and observation writers read."""
        e, b = self.env.env, self._buf
        k1 = e.nenvs if k1 is None else k1
        cfg, st = e.chunk_view(k0, k1)
        for key, _, field, _ in self._records:
            setattr(st, field, b[key][t, k0:k1].data_ptr())
        return cfg, st

    def _grad_state(self, t):
        """{'pp_state' | 'tj_state': an ic3_*_state whose recorded fields point at step t of the records} for
        ic3_bptt_step_io / ic3_ff_grad_io (a chunk's [K, ...] records start at its first step).  The other fields stay
        NULL: the backward reads none of them."""
        b = self._buf
        st = (_lib.TJState if self.is_tj else _lib.PPState)(**{field: b[key][t].data_ptr()
                                                               for key, _, field, _ in self._records})
        return {'tj_state' if self.is_tj else 'pp_state': C.pointer(st)}

    def _tj_record_obs(self, t, k0=0, k1=None):
        """[k1 - k0, N, O] traffic-junction observation of step t for env slots [k0, k1), written by ic3_tj_obs from the
        recorded env state into a new tensor (the torch backward keeps each step's observation until it has run)."""
        cfg, st = self._record_state(t, k0, k1)
        obs = torch.empty(cfg.B, self.args.nagents, self.env.observation_dim, device=self.env.env.device)
        _lib.check(_lib.load().ic3_tj_obs(C.byref(cfg), C.byref(st), obs.data_ptr(), _lib.stream()))
        return obs

    def _pp_sparse_obs(self, loc):
        """Non-zeros of the PP observation (predator_prey_env.py:188-210) as (index, value) pairs
        [R, 3*W*W] from a state snapshot loc [B, N+1, 2]."""
        e = self.env.env
        D, v, N = e.dim, e.vision, e.npredator
        NA = e.nagent_rows                                                   # + the prey's own row with enemy_comm
        W, V = 2 * v + 1, e.vocab_size
        loc = loc.long()
        pr, pc = loc[:, :N, 0], loc[:, :N, 1]
        ar = torch.arange(W, device=loc.device)
        dy, dx = ar.repeat_interleave(W), ar.repeat(W)                       # window cell w = dy*W + dx
        rr = loc[:, :NA, 0].unsqueeze(-1) - v + dy                           # [B, NA, W*W]
        cc = loc[:, :NA, 1].unsqueeze(-1) - v + dx
        inside = (rr >= 0) & (rr < D) & (cc >= 0) & (cc < D)
        base = torch.arange(W * W, device=loc.device) * V
        cls = torch.where(inside, rr * D + cc, torch.full_like(rr, D * D + 1)) + base
        npred = ((rr.unsqueeze(-1) == pr[:, None, None, :]) & (cc.unsqueeze(-1) == pc[:, None, None, :])).sum(-1)
        nprey = (rr == loc[:, N:, 0].unsqueeze(-1)) & (cc == loc[:, N:, 1].unsqueeze(-1))
        idx = torch.cat([cls, (base + V - 2).expand_as(cls), (base + V - 1).expand_as(cls)], -1)
        val = torch.cat([torch.ones_like(cls), nprey.long() * inside, npred * inside], -1).float()
        return idx.reshape(-1, 3 * W * W), val.reshape(-1, 3 * W * W)

    def _forward_window(self, t0, t1, h, c, adv, ret):
        """Differentiable re-run of steps [t0, t1) for all slots; returns (loss, h, c, stats)."""
        b, net, args = self._buf, self.policy_net, self.args
        B, N, H = self.env.env.nenvs, args.nagents, args.hid_size
        w = net._kernel_weights()
        w_e, b_e = w['enc_w'], w['enc_b']
        w_eT = None if self.is_tj else w_e.t().contiguous()
        loss = torch.zeros((), device=h.device)
        st = dict(action_loss=torch.zeros((), device=h.device), value_loss=torch.zeros((), device=h.device),
                  entropy=torch.zeros((), device=h.device))
        for t in range(t0, t1):
            keep = (1 - b['s_fresh'][t].float()).repeat_interleave(N).unsqueeze(1)        # trainer.py:50-51
            h, c = h * keep, c * keep
            if self.is_tj:
                x = F.linear(self._tj_record_obs(t).reshape(B * N, -1), w_e, b_e)         # comm.py:119
            else:
                idx, val = self._pp_sparse_obs(b['s_loc'][t])
                x = F.embedding_bag(idx, w_eT, per_sample_weights=val, mode='sum') + b_e
            fresh = b['s_fresh'][t].bool().unsqueeze(1)
            alive = torch.where(fresh, torch.ones_like(b['s_alive'][t]), b['s_alive'][t]).float()   # comm.py:99-112
            n_alive = alive.sum(1, keepdim=True)
            g = alive
            if self.hard:
                g = g * torch.where(fresh, torch.zeros_like(b['s_comm'][t]), b['s_comm'][t]).float()  # :171-175
            h, c, value, logps = policy_forward_torch(net, x, h, c, g, n_alive)
            value = value.view(B, N)
            alive_post = b['ralive'][t].float()
            act = b['action'][t].long()
            lp_taken = torch.zeros(B, N, device=h.device)
            ent = torch.zeros((), device=h.device)
            vmask = b['valid'][t].float().view(B, 1, 1)            # 0 for slots that already completed their batch
            for k, lp in enumerate(logps):
                lp = lp.view(B, N, -1)                                                     # comm.py:239
                lp_taken = lp_taken + lp.gather(-1, act[..., k:k + 1]).squeeze(-1)         # utils.py:42-46
                ent = ent - (lp * lp.exp() * vmask).sum()
            a_loss = (-adv[t] * lp_taken * alive_post).sum()                               # trainer.py:198-201
            v_loss = ((value - ret[t]).pow(2) * alive_post).sum()                          # :205-208
            step_loss = a_loss + args.value_coeff * v_loss
            if args.entr > 0:
                step_loss = step_loss - args.entr * ent                                    # :211-220
            loss = loss + step_loss
            st['action_loss'] += a_loss.detach(); st['value_loss'] += v_loss.detach(); st['entropy'] += ent.detach()
            det = (((b['s_tep'][t] + 1) % args.detach_gap) == 0).repeat_interleave(N).unsqueeze(1)   # trainer.py:56-60
            if bool(args.detach_gap <= self.args.max_steps):
                h = torch.where(det, h.detach(), h)
                c = torch.where(det, c.detach(), c)
        return loss, h, c, st

    LOSS_KEYS = ('action_loss', 'value_loss', 'entropy')

    def compute_grad(self, batch):
        """REINFORCE + value + entropy loss summed over every slot and step of the batch, gradients
        accumulated into ``p.grad`` (not yet divided by num_steps: train_batch does that,
        trainer.py:251-253).  Needs ``args.record_for_grad`` during the rollout.  Returns the reference's stat
        dict (trainer.py:222-225)."""
        v = self.compute_grad_device(batch).cpu().numpy()
        return {k: float(v[i]) for i, k in enumerate(self.LOSS_KEYS)}

    def compute_grad_device(self, batch):
        """compute_grad without a host synchronisation: the three loss sums come back as a float64 DEVICE vector
        (LOSS_KEYS order) so the data-parallel trainer can reduce them together with the batch statistics."""
        if not self.record_for_grad and not self.random_policy:
            raise RuntimeError("set args.record_for_grad = True before the rollout to use compute_grad")
        return self._losses_device()

    def _losses_device(self, K=None):
        """compute_grad_device after its check, with no host read, so a CUDA graph can hold it (update).  K: the
        kernels_ff chunk length (None: _ff_chunk_steps measures it now)."""
        b, args = self._buf, self.args
        e = self.env.env
        T, B, N = b['T'], e.nenvs, args.nagents
        ret = torch.empty(T, B, N, device=e.device)
        _lib.check(_lib.load().ic3_returns_scan(T, B, N, float(args.gamma), float(args.mean_ratio),
                                                b['reward'].data_ptr(), b['emask'].data_ptr(), b['mini'].data_ptr(),
                                                ret.data_ptr(), _lib.stream()))
        adv = ret - b['value'].view(T, B, N)                                               # trainer.py:176-177
        if args.normalize_rewards:                                   # :179-180, per slot, over its REAL steps only
            v = b['valid'].float().unsqueeze(-1)                     # [T, B, 1]
            cnt = v.sum(0, keepdim=True) * N
            mean = (adv * v).sum((0, 2), keepdim=True) / cnt
            var = (((adv - mean) * v) ** 2).sum((0, 2), keepdim=True) / (cnt - 1)      # torch.std: unbiased
            adv = (adv - mean) / var.sqrt()
        if self.random_policy:
            return self._random_losses(adv, ret)
        if self.grad_kernels:
            return self._compute_grad_kernels(adv, ret)
        if self.grad_ff:
            return self._compute_grad_ff(adv, ret, K)
        W = self.grad_window
        nw = (T + W - 1) // W
        dh = dc = None
        tot = torch.zeros(3, dtype=torch.float64, device=e.device)
        for k in reversed(range(nw)):
            t0, t1 = k * W, min(T, (k + 1) * W)
            h0 = b['ck_h'][k].clone().requires_grad_(True)
            c0 = b['ck_c'][k].clone().requires_grad_(True)
            loss, h1, c1, st = self._forward_window(t0, t1, h0, c0, adv, ret)
            if dh is not None:                     # gradient arriving from the later window
                loss = loss + (h1 * dh).sum() + (c1 * dc).sum()
            loss.backward()
            # variants without a cell state / without a carried hidden state leave these gradients undefined: zero
            dh = h0.grad.detach() if h0.grad is not None else torch.zeros_like(h0)
            dc = c0.grad.detach() if c0.grad is not None else torch.zeros_like(c0)
            tot += torch.stack([st[key] for key in self.LOSS_KEYS]).double()
        return tot

    def _random_losses(self, adv, ret):
        """compute_grad of models.Random (trainer.py:186-220): the three loss sums straight from the records, in float64;
        no forward to re-run and no parameter to reach (Random's outputs are leaves of the graph)."""
        b, args = self._buf, self.args
        T, B, N = b['T'], self.env.env.nenvs, args.nagents
        heads = list(args.naction_heads)
        off = torch.tensor([sum(heads[:k]) for k in range(len(heads))], device=adv.device)
        logp = b['logp'].double()                                                    # [T, B, N, sum(na)]
        lp = logp.gather(-1, b['action'].long() + off).sum(-1)                       # utils.py:42-46
        alive = b['ralive'].double()
        ret = ret.double()
        a_loss = (-adv.double() * lp * alive).sum()                                  # trainer.py:198-201
        v_loss = ((b['value'].view(T, B, N).double() - ret) ** 2 * alive).sum()      # :205-208
        ent = -(logp * logp.exp() * b['valid'].double().view(T, B, 1, 1)).sum()      # :213-217, real steps only
        return torch.stack([a_loss, v_loss, ent])

    def _compute_grad_kernels(self, adv, ret):
        """Hand-written BPTT (csrc/bptt_tc.cu): one ic3_bptt_step per lock-step iteration, last to first, after
        ic3_bptt_begin_dev has reduced max |c| of the record, the bound behind the operand scale, on the device.  In
        window mode (record_mode) the policy step re-runs each window from its checkpoint just ahead of the backward
        (_recompute_window); the gradient is bit-identical to full records'.  Returns the device float64 vector of the
        three loss sums."""
        b, net, args, e = self._buf, self.policy_net, self.args, self.env.env
        lib = _lib.load()
        T, B, N, H = b['T'], e.nenvs, args.nagents, args.hid_size
        s = _lib.stream()
        cfg = self._policy_cfg()
        w = net.packed()
        hc = not self._h_only_records()        # the tanh RNN: h alone, no encoder table (x is no operand of its GEMMs)
        plan = self._bptt_plan(cfg, w, _lib.ptr(self._encoder_table()) if hc else None)
        if self._bptt is None or self._bptt['B'] != B:
            nbytes = int(lib.ic3_bptt_workspace_bytes(C.byref(plan)))
            if nbytes == 0:
                raise NotImplementedError("this configuration is outside the BPTT kernels (use grad_impl='autograd')")
            self._bptt = dict(B=B, ws=torch.empty(nbytes, dtype=torch.uint8, device=e.device),
                              dh=torch.zeros(B * N, H, device=e.device),
                              dc=torch.zeros(B * N, H, device=e.device) if hc else None,
                              losses=torch.zeros(3, dtype=torch.float64, device=e.device))
        st = self._bptt
        plan.workspace = st['ws'].data_ptr()
        adv = adv.contiguous()
        cut = None
        if args.detach_gap <= args.max_steps:                                  # trainer.py:56-60
            cut = (((b['s_tep'] + 1) % args.detach_gap) == 0).to(torch.uint8).contiguous()
        window = self._record_mode == 'window'
        W, nb = self.grad_window, self._window_buffers()
        # max |c| over every step's c, from the full record or from the per-step maxima the rollout kept in window mode;
        # the tanh RNN has no cell state, and its operand scale bounds |dh| alone
        csrc = None if not hc else b['c_abs'] if window else b['rec_c'][1:]

        def state(t):                          # (h, c) entering step t and h' leaving it (c: None for the tanh RNN)
            if not window:
                return b['rec_h'][t], b['rec_c'][t] if hc else None, b['rec_h'][t + 1]
            k, j = divmod(t, W)                # window mode: in the window buffers, entered from checkpoint k
            wh = b['win_h'][k % nb]
            if j == 0:
                return b['ck_h'][k], b['ck_c'][k] if hc else None, wh[0]
            return wh[j - 1], b['win_c'][k % nb][j - 1] if hc else None, wh[j]
        # window mode: window k, steps [t0, t1), is re-run on this stream right before ic3_bptt_step(t1 + 1) is issued
        # (before ic3_bptt_begin_dev when there is no such step).  The look-ahead ic3_bptt_prepare(t) on the library's side
        # stream waits for this stream's work up to ic3_bptt_step(t + 2), so it sees every window it reads; and the
        # buffer window k overwrites (that of window k + nb, all of whose steps are >= t1 + 2) has no reader left.
        todo = list(reversed(range((T + W - 1) // W))) if window else []

        def recompute_due(t):
            while todo and min(T, (todo[0] + 1) * W) + 1 >= t:
                self._recompute_window(todo.pop(0))

        recompute_due(T)
        st['dh'].zero_()
        if hc:
            st['dc'].zero_()
        _lib.check(lib.ic3_bptt_begin_dev(C.byref(plan), _lib.ptr(csrc), 0 if csrc is None else csrc.numel(), s))
        value = b['value']

        def step_io(t):
            hp, cp, hn = state(t)
            return _lib.BpttStepIO(t=t, h_prev=hp.data_ptr(), c_prev=_lib.ptr(cp),
                                   h_new=hn.data_ptr(), fresh=b['s_fresh'][t].data_ptr(),
                                   comm=b['s_comm'][t].data_ptr() if self.hard else None,
                                   alive=b['s_alive'][t].data_ptr(), cut=cut[t].data_ptr() if cut is not None else None,
                                   logp=b['logp'][t].data_ptr(), action=b['action'][t].data_ptr(),
                                   value=value[t].data_ptr(), ret=ret[t].data_ptr(), adv=adv[t].data_ptr(),
                                   alive_post=b['ralive'][t].data_ptr(), valid=b['valid'][t].data_ptr(),
                                   dh=st['dh'].data_ptr(), dc=_lib.ptr(st['dc']), err=b['err'].data_ptr(),
                                   **self._grad_state(t))
        # look-ahead: the heads gradient and the operand images of step t - 1 do not depend on the recursion; they are
        # launched on the library's side stream before step t and overlap its tensor-core kernels
        nxt = step_io(T - 1) if T > 0 else None
        if nxt is not None:
            _lib.check(lib.ic3_bptt_prepare(C.byref(plan), C.byref(nxt), s))
        for t in reversed(range(T)):
            recompute_due(t)
            io = nxt
            if t > 0:
                nxt = step_io(t - 1)
                _lib.check(lib.ic3_bptt_prepare(C.byref(plan), C.byref(nxt), s))
            _lib.check(lib.ic3_bptt_step(C.byref(plan), C.byref(io), s))
        # parameter gradients are ADDED to the .grad buffers (flat views of FlatRMSprop)
        params, grads = self._param_structs()
        _lib.check(lib.ic3_bptt_finish(C.byref(plan), C.byref(params), C.byref(grads), st['losses'].data_ptr(), s))
        return st['losses']

    # Lock-steps per chunk of the non-recurrent kernels: as many as the memory the device has left holds (measured like
    # the BPTT records in _pick_record_mode), at most FF_CHUNK_ROWS agent rows (2^21: 25 steps, about 10 GB of workspace
    # at predator-prey hard with 8192 slots and 2 passes; one step of that size already fills the card many times
    # over), and at most FF_CHUNK_STEPS steps when set
    FF_CHUNK_ROWS = 1 << 21
    FF_CHUNK_STEPS = None

    def _ff_plan(self, cfg, w, rows, workspace=None):
        e, args = self.env.env, self.args
        return _lib.FfGradPlan(cfg=C.pointer(cfg), w=None if w is None else C.pointer(w),
                               pp_env=None if self.is_tj else C.pointer(e.cfg), tj_env=C.pointer(e.cfg) if self.is_tj else None,
                               value_coeff=float(args.value_coeff), entr=float(args.entr), max_rows=rows,
                               workspace=workspace)

    def _ff_chunk_steps(self, T, cfg):
        """Lock-steps per chunk K of ic3_ff_grad_chunk for a T-step rollout: what the workspace of K steps needs must fit
        in the device's free memory plus the allocator's unused reserve, minus RECORD_MARGIN_BYTES; K * B * N is at most
        FF_CHUNK_ROWS (at least one step).  A resumed run keeps the K its last update used (ff_chunk_pin)."""
        if self.ff_chunk_pin is not None:
            return int(self.ff_chunk_pin)
        e = self.env.env
        lib = _lib.load()
        rows = e.nenvs * self.args.nagents
        nbytes = lambda k: int(lib.ic3_ff_grad_workspace_bytes(C.byref(self._ff_plan(cfg, None, k * rows))))
        one = nbytes(1)
        per_step = max(1, nbytes(2) - one)
        free = self._device_bytes_free()
        k = max(1, min(T, (free - self.RECORD_MARGIN_BYTES - one) // per_step + 1, self.FF_CHUNK_ROWS // rows))
        if self.FF_CHUNK_STEPS is not None:
            k = max(1, min(k, int(self.FF_CHUNK_STEPS)))
        return int(k)

    def _compute_grad_ff(self, adv, ret, K=None):
        """grad_impl 'kernels_ff' (ic3_ff_grad_*): the rollout's T lock-steps in chunks of K consecutive steps, each one
        batch of K*B env slots (records are [T, B, ...]), in any order since no state crosses a step; the backward's
        products run on the tensor cores.  K: None = _ff_chunk_steps.  Returns the device float64 vector of the three
        loss sums."""
        b, net, args, e = self._buf, self.policy_net, self.args, self.env.env
        lib = _lib.load()
        T, B, N = b['T'], e.nenvs, args.nagents
        s = _lib.stream()
        cfg = self._policy_cfg()
        w = net.packed()
        if K is None:
            K = self._ff_chunk_steps(T, cfg)
        plan = self._ff_plan(cfg, w, K * B * N)
        nbytes = int(lib.ic3_ff_grad_workspace_bytes(C.byref(plan)))
        if nbytes == 0:
            raise NotImplementedError("this configuration is outside the non-recurrent gradient kernels")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=e.device)     # stream-ordered: freed after the kernels ran
        plan.workspace = ws.data_ptr()
        losses = torch.zeros(3, dtype=torch.float64, device=e.device)
        adv = adv.contiguous()
        _lib.check(lib.ic3_ff_grad_begin(C.byref(plan), s))
        for t in range(0, T, K):
            io = _lib.FfGradIO(nsteps=min(K, T - t), fresh=b['s_fresh'][t].data_ptr(),
                               comm=b['s_comm'][t].data_ptr() if self.hard else None, alive=b['s_alive'][t].data_ptr(),
                               logp=b['logp'][t].data_ptr(), action=b['action'][t].data_ptr(),
                               value=b['value'][t].data_ptr(), ret=ret[t].data_ptr(), adv=adv[t].data_ptr(),
                               alive_post=b['ralive'][t].data_ptr(), valid=b['valid'][t].data_ptr(),
                               **self._grad_state(t))
            _lib.check(lib.ic3_ff_grad_chunk(C.byref(plan), C.byref(io), s))
        params, grads = self._param_structs()
        _lib.check(lib.ic3_ff_grad_finish(C.byref(plan), C.byref(params), C.byref(grads), losses.data_ptr(), s))
        self.ff_chunk_steps = K
        return losses

    def _recompute_window(self, k):
        """Window mode: re-run the policy step over steps [k W, min(T, (k+1) W)) from checkpoint k into the window
        buffer k % nb on the current stream; returns its (h, c) views [steps, B*N, H], row j = (h', c') of step k W + j.
        Inputs come from the per-step records (fresh / comm / alive, and x from the recorded env state through the
        fused index encoder with the per-position table); nothing is sampled and value / log-probs go to scratch.  The
        tensor-core policy step is deterministic and every encoder form gives the same x, so each row equals the
        rollout's (h', c') bit for bit -- except for slots that had already completed their batch (valid = 0), whose
        inputs the env step no longer records; those rows carry no loss and no gradient.
        The tanh RNN (h alone, c is None): the index encoder from the recorded env state into the rollout's x buffer,
        then the policy step of the rollout's policy_impl ('simt', or 'tc_tanh': the recurrent form of ff_tc_kernel; the
        policy's packed weights and workspace select it, as in _enqueue), the same kernels and operands as the rollout."""
        b, e, net = self._buf, self.env.env, self.policy_net
        lib = _lib.load()
        B, W = e.nenvs, self.grad_window
        t0, t1 = k * W, min(b['T'], (k + 1) * W)
        cfg = self._policy_cfg()
        w = net.packed()
        nb = self._window_buffers()
        s = _lib.stream()
        hc = not self._h_only_records()
        wh, wc = b['win_h'][k % nb], b['win_c'][k % nb] if hc else None
        table = self._encoder_table() if hc else None
        enc = lib.ic3_tj_encoder_index if self.is_tj else lib.ic3_pp_encoder_index
        ws, _ = net.workspace(B)
        for t in range(t0, t1):
            j = t - t0
            hin = b['ck_h'][k] if j == 0 else wh[j - 1]
            cin = None if not hc else b['ck_c'][k] if j == 0 else wc[j - 1]
            ecfg, est = self._record_state(t)          # held until the policy step below has read them
            if hc:       # the fused index encoder with the per-position table
                src = dict(_lib.env_source(ecfg, est), x=None, x_table=table.data_ptr())
            else:        # the index encoder into the rollout's x buffer
                _lib.check(enc(C.byref(ecfg), C.byref(est), C.byref(cfg), C.byref(w), b['x'].data_ptr(), s))
                src = dict(x=b['x'].data_ptr())
            io = _lib.PolicyIO(h=hin.data_ptr(), c=_lib.ptr(cin),
                               comm_action=b['s_comm'][t].data_ptr() if self.hard else None,
                               alive=b['s_alive'][t].data_ptr(), fresh=b['s_fresh'][t].data_ptr(), tick=None,
                               draws=None, h_out=wh[j].data_ptr(), c_out=wc[j].data_ptr() if hc else None,
                               value=b['win_value'].data_ptr(), logp=b['win_logp'].data_ptr(), action=None,
                               workspace=_lib.ptr(ws), err=b['err'].data_ptr(), **src)
            _lib.check(lib.ic3_policy_step(C.byref(cfg), C.byref(w), C.byref(io), s))
        return wh[:t1 - t0], wc[:t1 - t0] if hc else None

    def _param_structs(self):
        """ic3_policy_params of the parameters and of their gradient buffers (reference layouts), by kernel role."""
        net = self.policy_net
        scratch = self.__dict__.setdefault('_grad_scratch', {})

        def grad_ptr(p):
            if isinstance(p, torch.nn.Parameter):
                if p.grad is None:
                    p.grad = torch.zeros_like(p)
                return p.grad.data_ptr()
            key = p.data_ptr()                       # frozen buffer (models.py: zero comm projection): discard its gradient
            if key not in scratch:
                scratch[key] = torch.zeros_like(p)
            return scratch[key].data_ptr()

        return net.policy_params(lambda p: p.data_ptr()), net.policy_params(grad_ptr)

    # only used when there is a single process (trainer.py:245-256)
    def train_batch(self, epoch):
        return self.update(epoch)

    # ------------------------------------------------------------------ the update
    # head: gradient zeroing, rollout, returns, advantages, gradient kernels and their finish, then ic3_stat_reduce (after
    # the gradient, so its flag word also holds what the gradient kernels set), into the float64 vector out = [statistics
    # | loss sums | optimizer flags].  tail: RMSprop with the divisor read from out (ic3_rmsprop_step_dev skips it on
    # error flags), then the weight pack and encoder table the next rollout reads.  Neither reads back to the host, so
    # graph_update can replay them: one graph, or one each around a reduce.  models.Random has no gradient to zero and no
    # tail: its .grad stays None and the optimizer state empty, as the reference's step skips it (trainer.py:251-254).

    def _update_head(self, rollout, K):
        b = self._buf
        if not self.random_policy:
            self.optimizer.zero_grad(set_to_none=False)
            b['opt_err'].zero_()
        rollout()
        losses = self._losses_device(K)
        vec = self.stat_vector()
        return torch.cat([vec, losses.to(vec.dtype), torch.zeros(1, dtype=vec.dtype, device=vec.device)])

    def _update_tail(self, out):
        b = self._buf
        self.optimizer.step_dev(out, b['opt_err'])
        out[-1:].copy_(b['opt_err'])
        self._refresh_weights(b, self.env.env, force=True)

    def update(self, epoch, reduce=None):
        """One training update (trainer.py:245-256): rollout, gradient and RMSprop step, with one host read.  reduce(out),
        if given, runs eagerly between the head and the tail (the data-parallel all-reduces of the flat gradients and of
        out, in place).  graph_update: head and tail are replayed from CUDA graphs; otherwise they run eagerly, the
        rollout replayed from its own graph with use_graph (as run_batch does).  Raises on a device error flag of the
        rollout or the gradient, in which case the parameters and the optimizer state are as they were.  Returns the
        stat dict."""
        if not self.record_for_grad and not self.random_policy:
            raise RuntimeError("set args.record_for_grad = True before the rollout to use compute_grad")
        net, opt = self.policy_net, self.optimizer
        learns = not self.random_policy
        T, quota = self.batch_plan()
        b, e = self._begin(T, epoch)
        if learns and 'opt_err' not in b:
            b['opt_err'] = torch.zeros(1, dtype=torch.int32, device=e.device)
        key = lambda: self._graph_key(T, e, int(quota), self._record_mode, self._ff_K, opt.lr, opt.alpha, opt.eps)
        K = None                             # kernels_ff chunk length: measured for each update and each capture
        if self.grad_ff:
            held = self.graph_update and self._graphs.get('update', (None,))[0] == key()
            K = self._ff_K if held else self._ff_chunk_steps(T, self._policy_cfg())
        if self.graph_update:
            self._ff_K = K                   # part of the key: a captured update keeps the K it holds
            # the warm-up before the capture also rewinds the parameters, gradients and second moments
            head = lambda: self._update_head(lambda: self._enqueue(T, quota), K)
            out, captured = self._replay('update', key(), b, e, (head, self._update_tail), reduce,
                                         (opt.flat_params, opt.flat_grads, opt.flat_square_avg))
            self.update_captures += captured
        else:
            out = self._update_head(lambda: self._run_rollout(T, quota, b, e), K)
            if reduce is not None:
                reduce(out)
            if learns:
                self._update_tail(out)
        host = out.cpu().numpy()
        nstat = host.size - 4
        stat = self.stat_from_vector(host[:nstat])    # raises on the flags; the tail then changed nothing
        if int(host[-1]):
            raise RuntimeError("device-side error flag %#x in the optimizer step (step count %r)" % (int(host[-1]),
                                                                                                host[1]))
        if learns:
            opt.steps += 1
            opt.mark_params_changed()
            net.mark_packed_current([] if 'obs' in b else [e])      # the tables _update_tail re-built (_refresh_weights)
        if self.grad_ff:
            self.ff_chunk_steps = K
        merge_stat({k: float(host[nstat + i]) for i, k in enumerate(self.LOSS_KEYS)}, stat)
        self.stats = stat
        return stat

    def state_dict(self):
        return self.optimizer.state_dict()

    def load_state_dict(self, state):
        self.optimizer.load_state_dict(state)

    # ------------------------------------------------------------------ run state (resuming a run)
    # What crosses an update boundary besides the parameters and the RMSprop state of state_dict: the env's device state
    # (its tick / episode counters key the Philox streams), the traffic-junction curriculum, the evaluation env once it
    # exists, and the kernels_ff chunk length K (gradients for different K differ in the last bits).  Graph caches are
    # not state: the first update after a load captures anew.

    def run_fingerprint(self):
        """What shapes the run, as plain values: load_run_state refuses a state taken under other values."""
        a, e = self.args, self.env.env
        dist = torch.distributed
        fp = {k: getattr(a, k, None) for k in RUN_FINGERPRINT_ARGS}
        fp.update(world=dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1,
                  nenvs=e.nenvs, eval_nenvs=int(getattr(a, 'eval_nenvs', None) or e.nenvs), seed=int(getattr(a, 'seed', 0)),
                  grad_impl=self.grad_impl, policy_impl=getattr(self.policy_net, 'policy_impl', None),
                  use_graph=self.use_graph, graph_update=self.graph_update)
        return fp

    def run_state(self):
        """{'fingerprint': run_fingerprint(), 'ranks': [this process's state]} on the host; load_run_state takes it."""
        return dict(fingerprint=self.run_fingerprint(), ranks=[self.rank_state()])

    def load_run_state(self, state):
        """Continue the run that run_state() was taken from (the parameters and the optimizer come from state_dict).
        Refuses, before touching the device, a state whose fingerprint differs from this trainer's."""
        check_fingerprint(state['fingerprint'], self.run_fingerprint())
        if len(state['ranks']) != 1:
            raise ValueError("the run state holds %d ranks; MultiGPUTrainer.load_run_state takes it" % len(state['ranks']))
        self.load_rank_state(state['ranks'][0])

    def rank_state(self):
        """This process's part of the run state: its training env, its evaluation env (None before the first
        evaluation) and the kernels_ff chunk length of the last update (None for other gradients)."""
        ev = getattr(self, '_eval', None)
        return dict(env=self._env_state(self.env.env), eval=None if ev is None else self._env_state(ev['env']),
                    ff_chunk_steps=getattr(self, 'ff_chunk_steps', None) if self.grad_ff else None)

    def load_rank_state(self, d):
        self._load_env_state(self.env.env, d['env'])
        if d['eval'] is not None:
            self._load_env_state(self._eval_state()['env'], d['eval'])
        self.ff_chunk_pin = d['ff_chunk_steps']

    def _env_state(self, e):
        d = dict(device={k: v.cpu() for k, v in zip(e._STATE, e.snapshot())})
        if self.is_tj:
            d.update(exact_rate=e.exact_rate, add_rate=e.add_rate, epoch_last_update=e.epoch_last_update)
        return d

    def _load_env_state(self, e, d):
        snap = []
        for k in e._STATE:
            live, v = getattr(e, k), d['device'][k]
            if v.shape != live.shape or v.dtype != live.dtype:
                raise ValueError("run state field %s is %s %s, the env holds %s %s" % (k, v.dtype, tuple(v.shape),
                                                                                       live.dtype, tuple(live.shape)))
            snap.append(v.to(live.device))
        e.restore(snap)
        if self.is_tj:
            e.exact_rate, e.add_rate, e.epoch_last_update = d['exact_rate'], d['add_rate'], d['epoch_last_update']
            e.cfg.spawn_thr = e._spawn_thr()


# The arguments of a run's fingerprint besides those Trainer.run_fingerprint resolves: env and geometry, policy, loss
# and optimizer, and the loop (a missing one reads None)
RUN_FINGERPRINT_ARGS = (
    'env_name', 'nagents', 'dim', 'vision', 'mode', 'nenemies', 'enemy_comm', 'no_stay', 'moving_prey', 'difficulty',
    'vocab_type', 'add_rate_min', 'add_rate_max', 'curr_start', 'curr_end',
    'commnet', 'random', 'recurrent', 'rnn_type', 'hid_size', 'hard_attn', 'comm_mode', 'comm_passes', 'comm_mask_zero',
    'comm_action_one', 'share_weights', 'mean_ratio', 'detach_gap', 'obs_mode', 'forward_grad',
    'gamma', 'lrate', 'entr', 'value_coeff', 'normalize_rewards', 'grad_window',
    'batch_size', 'max_steps', 'batch_boundary', 'epoch_size', 'rollout_only')


def check_fingerprint(stored, current):
    """Raise ValueError naming every field whose stored value differs from the current one."""
    diff = ['%s (stored %r, now %r)' % (k, stored.get(k), current.get(k))
            for k in sorted(set(stored) | set(current)) if stored.get(k) != current.get(k)]
    if diff:
        raise ValueError("the run state belongs to another configuration: " + ', '.join(diff) +
                         "; a run resumes only under the configuration it started with")
