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
"""
import ctypes as C
import math
from collections import namedtuple

import torch
import torch.nn.functional as F

from . import _lib
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
        self._bptt = None
        self._buf = None
        self._record_mode = None             # 'full' | 'window' per allocation (record_mode)
        self._graph = None
        self._graph_key = None
        self._side = None                    # stream of the dense observation writer (_overlap_obs)
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

    def _policy_cfg(self):
        """ic3_policy_cfg of the policy step over this GPU's slots, with the env's Philox key and env ids."""
        e = self.env.env
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

    def _encoder_table(self, cfg=None, w=None):
        """The policy's per-position encoder table for this environment (CommNetMLP.encoder_table), built from its
        current packed weights; cfg and w are accepted for callers that hold them and are not needed."""
        return self.policy_net.encoder_table(self.env.env)

    # ------------------------------------------------------------------ buffers
    def _alloc(self, T):
        self._buf = self._graph = None       # the previous buffers go back to the allocator before the records are sized
        e = self.env.env
        B, N, H = e.nenvs, self.args.nagents, self.args.hid_size
        dev = e.device
        nh = len(self.args.naction_heads)
        A = sum(self.args.naction_heads)
        z = lambda *s, dtype=torch.float32: torch.zeros(*s, dtype=dtype, device=dev)
        b = dict(T=T, comm=z(B, N, dtype=torch.uint8), alive=torch.ones(B, N, dtype=torch.uint8, device=dev),
                 fresh=torch.ones(B, dtype=torch.uint8, device=dev), t_ep=z(B, dtype=torch.int32),
                 action=z(T, B, N, nh, dtype=torch.int32), logp=z(T, B, N, A), value=z(T, B * N),
                 reward=z(T, B, N), emask=z(T, B, dtype=torch.uint8), mini=z(T, B, N, dtype=torch.uint8),
                 ralive=z(T, B, N, dtype=torch.uint8), step_reward=z(B, N),
                 stat_reward=z(B, N), stat_comm=z(B, N), stat_success=z(B, dtype=torch.int32),
                 stat_episodes=z(B, dtype=torch.int32), stat_steps=z(B, dtype=torch.int32),
                 err=z(1, dtype=torch.int32), halted=z(B, dtype=torch.uint8), valid=z(T, B, dtype=torch.uint8),
                 statvec=z(4 + 2 * N, dtype=torch.float64))
        if self.random_policy:                # no encoder, observation or recurrent state
            self._buf = b
            return b
        b.update(h=z(B * N, H), c=z(B * N, H), x=z(B * N, H))
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
        self._graph = None
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

    def _overlap_obs(self):
        """Dense observations on the tensor-core policy path: the policy step computes x from the env state (the fused
        index encoder; without the per-position table, which measured no faster beside the writer, so dense mode never
        builds it) and the observation block is written concurrently on a side stream.  Not for blocks smaller than
        OVERLAP_MIN_OBS_BYTES."""
        if self.obs_mode != 'dense':
            return False
        e = self.env.env
        if e.nenvs * self.args.nagents * self.env.observation_dim * 4 < self.OVERLAP_MIN_OBS_BYTES:
            return False
        return self.policy_net.fuses_encoder(e)

    def _enqueue(self, T, quota=0):
        """Enqueue T lock-step iterations on the current stream (no host sync).  quota > 0: reference batch
        boundary -- a slot halts at the first episode end with >= quota steps (ic3_rollout_io.batch_size);
        quota = 0: episodes still open at iteration T-1 are cut there."""
        if self.random_policy:
            return self._enqueue_random(T, quota)
        b, e, net = self._buf, self.env.env, self.policy_net
        lib = _lib.load()
        B = e.nenvs
        cfg = self._policy_cfg()
        w = net.packed()
        s = _lib.stream()
        ws, _ = net.workspace(B)          # tensor-core path scratch (None for the fp32 SIMT kernel)
        rec = self.record_for_grad
        full = rec and self._record_mode == 'full'    # the policy step writes (h, c) straight into the records
        window = rec and self._record_mode == 'window'    # (h, c) checkpoints + max |c| per step (_alloc)
        hc = not self._h_only_records()               # the tanh RNN's kernel records: h alone
        dense = self.obs_mode == 'dense'
        # dense observations written on a side stream while the policy step runs (see _overlap_obs)
        overlap = self._overlap_obs()
        # tensor-core path: the index encoder is fused into the policy step (x never leaves the operand image)
        fused_x = self._fused_x() or overlap
        src = {}
        if fused_x:
            src = dict(_lib.env_source(e.cfg, e.state), x_table=None if overlap else _lib.ptr(self._encoder_table()))
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
            io = _lib.PolicyIO(x=None if fused_x else b['x'].data_ptr(), h=hin.data_ptr(), c=cin.data_ptr(),
                               comm_action=b['comm'].data_ptr() if self.hard else None, alive=b['alive'].data_ptr(),
                               fresh=b['fresh'].data_ptr(), tick=e.tick.data_ptr(), draws=None,
                               h_out=hout.data_ptr(), c_out=cout.data_ptr(), value=b['value'][t].data_ptr(),
                               logp=b['logp'][t].data_ptr(), action=b['action'][t].data_ptr(),
                               workspace=_lib.ptr(ws), err=b['err'].data_ptr(), **src)
            _lib.check(lib.ic3_policy_step(C.byref(cfg), C.byref(w), C.byref(io), s))
            if window and hc:
                # max |c'| of this step: the backward's operand scale needs the bound over every step's c before it
                # re-runs any window, the same value a full record gives (_compute_grad_kernels)
                torch.linalg.vector_norm(b['c'], math.inf, out=b['c_abs'][t])
            if overlap:
                main.wait_stream(side)
            self._env_step(t, T, quota, snap, s)

    def _env_step(self, t, T, quota, snap, s):
        """Env step of lock-step iteration t on the actions the policy step wrote to the records, with the
        Trainer.get_episode bookkeeping and auto-reset (ic3_rollout_io; ``snap``: its snap_* fields)."""
        b, e, args = self._buf, self.env.env, self.args
        lib = _lib.load()
        nh = len(args.naction_heads)
        r = _lib.RolloutIO(t=t, max_steps=args.max_steps, nheads=nh, hard_attn=int(self.hard),
                           comm_action_one=int(bool(args.comm_action_one)),
                           last=int(t == T - 1 and quota <= 0), batch_size=int(quota),
                           halted=b['halted'].data_ptr(), rec_valid=b['valid'].data_ptr(), **snap,
                           action=b['action'][t].data_ptr(), t_ep=b['t_ep'].data_ptr(),
                           fresh=b['fresh'].data_ptr(), comm_next=b['comm'].data_ptr(),
                           alive_next=b['alive'].data_ptr(), rec_reward=b['reward'].data_ptr(),
                           rec_episode_mask=b['emask'].data_ptr(), rec_mini_mask=b['mini'].data_ptr(),
                           rec_alive=b['ralive'].data_ptr(), stat_reward=b['stat_reward'].data_ptr(),
                           stat_comm=b['stat_comm'].data_ptr(), stat_success=b['stat_success'].data_ptr(),
                           stat_episodes=b['stat_episodes'].data_ptr(), stat_steps=b['stat_steps'].data_ptr())
        if self.is_tj:
            _lib.check(lib.ic3_tj_step(C.byref(e.cfg), C.byref(e.state), b['action'][t].data_ptr(), nh, None,
                                       b['step_reward'].data_ptr(), None, b['err'].data_ptr(), C.byref(r), s))
        else:
            _lib.check(lib.ic3_pp_step(C.byref(e.cfg), C.byref(e.state), b['action'][t].data_ptr(), nh,
                                       b['step_reward'].data_ptr(), None, b['err'].data_ptr(), C.byref(r), s))

    def random_cfg(self):
        """ic3_policy_cfg of the Random policy step: the fields ic3_random_policy_step reads (B, N, heads, Philox key
        and env ids of this GPU's slots)."""
        e, heads = self.env.env, list(self.args.naction_heads)
        return _lib.PolicyCfg(B=e.nenvs, N=self.args.nagents, nheads=len(heads),
                              head_dim=(C.c_int32 * _lib.MAX_HEADS)(*heads), env_id0=e.cfg.env_id0, seed=e.cfg.seed)

    def _enqueue_random(self, T, quota):
        """_enqueue for models.Random: per lock-step iteration one ic3_random_policy_step (value, log-probs and actions
        into the records, from the env's action tick) and the env step."""
        b, e = self._buf, self.env.env
        lib = _lib.load()
        cfg = self.random_cfg()
        s = _lib.stream()
        for t in range(T):
            io = _lib.PolicyIO(tick=e.tick.data_ptr(), value=b['value'][t].data_ptr(), logp=b['logp'][t].data_ptr(),
                               action=b['action'][t].data_ptr())
            _lib.check(lib.ic3_random_policy_step(C.byref(cfg), C.byref(io), None, s))
            self._env_step(t, T, quota, {}, s)

    def _episode_boundary(self, epoch):
        e, b = self.env.env, self._buf
        if self.is_tj:
            e.reset(epoch, want_obs=False)
        else:
            e.reset(want_obs=False)
        for k in ('stat_reward', 'stat_comm', 'stat_success', 'stat_episodes', 'stat_steps', 't_ep', 'halted'):
            b[k].zero_()
        b['fresh'].fill_(1)

    def rollout(self, T, epoch=0, quota=0):
        """T lock-step iterations from fresh episodes in every slot (``quota``: see _enqueue).  Returns a
        RolloutBatch of stacked [T, B, ...] device tensors (views of the trainer's record buffers)."""
        e = self.env.env
        if self._buf is None or self._buf['T'] != T:
            self._alloc(T)
        b = self._buf
        self._episode_boundary(epoch)             # trainer.py:28-32, 45-51
        b['err'].zero_()
        if not self.random_policy:
            self.policy_net.packed()              # (re)pack weights outside any graph capture
            if self._fused_x():
                self._encoder_table()             # ... and the encoder table with them
        if self.use_graph:
            # kernel arguments passed BY VALUE are frozen into a captured graph: everything of that kind that can
            # change between rollouts is part of the key (the TJ curriculum moves cfg.spawn_thr, traffic_junction_env.py:
            # 196-200,620-626; a re-seeded env changes cfg.seed) and a stale graph is re-captured
            key = (T, int(quota), int(getattr(e.cfg, 'spawn_thr', 0)), int(e.cfg.seed), int(e.cfg.env_id0))
            if self._graph is None or self._graph_key != key:
                # warm-up pass (lazy function attributes, allocator) on a snapshot of the env state, rewound afterwards:
                # the captured pass then starts from exactly the state an eager rollout would start from (same RNG ticks)
                snap = e.snapshot()
                keys = ('fresh', 'comm', 'alive', 't_ep', 'h', 'c', 'halted', 'stat_reward', 'stat_comm', 'stat_success',
                        'stat_episodes', 'stat_steps')
                saved = {k: b[k].clone() for k in keys if k in b}
                self._enqueue(T, quota)
                torch.cuda.synchronize()
                e.restore(snap)                   # env state, RNG ticks ...
                for k, v in saved.items():        # ... and the trainer-side episode state, as the boundary above left them
                    b[k].copy_(v)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._enqueue(T, quota)
                self._graph, self._graph_key = g, key
                g.replay()
            else:
                self._graph.replay()
        else:
            self._enqueue(T, quota)
        return RolloutBatch(action=b['action'], logp=b['logp'], value=b['value'].view(T, e.nenvs, -1),
                            reward=b['reward'], episode_mask=b['emask'], episode_mini_mask=b['mini'],
                            alive_mask=b['ralive'], valid=b['valid'])

    def stat_vector(self):
        """Device float64 vector [num_episodes, num_steps, success, err flags, reward[N], comm_action[N]] of this
        GPU's slots (one kernel, csrc/returns.cu ic3_stat_reduce); no host synchronisation."""
        b, e = self._buf, self.env.env
        _lib.check(_lib.load().ic3_stat_reduce(e.nenvs, self.args.nagents, b['stat_episodes'].data_ptr(),
                                               b['stat_steps'].data_ptr(), b['stat_success'].data_ptr(),
                                               b['err'].data_ptr(), b['stat_reward'].data_ptr(),
                                               b['stat_comm'].data_ptr() if self.hard else None,
                                               b['statvec'].data_ptr(), _lib.stream()))
        return b['statvec']

    def stat_from_vector(self, v):
        """Host-side stat dict with the reference's keys (trainer.py:73-75,86-88,109-110,124-125,235) from a
        stat_vector() (of this GPU, or summed over ranks) that has been copied to the host."""
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
            stat['add_rate'] = self.env.env.add_rate * stat['num_episodes']
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
            return self._compute_grad_ff(adv, ret)
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
        """Hand-written BPTT (csrc/bptt_tc.cu): one ic3_bptt_step per lock-step iteration, last to first (one host read
        up front: max |c| of the record, the bound behind the operand scale).  In window mode (record_mode) the policy
        step re-runs each window from its checkpoint just ahead of the backward (_recompute_window); the gradient is
        bit-identical to full records'.  Returns the device float64 vector of the three loss sums."""
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
        if not hc:
            cmax = 0.0                          # no cell state: the operand scale bounds |dh| alone
        elif window:
            cmax = float(b['c_abs'].max().item())                              # tracked per step by the rollout
        else:
            lo, hi = torch.aminmax(b['rec_c'][1:])                              # bound of |c| for the operand scale
            cmax = max(abs(float(lo.item())), abs(float(hi.item())))

        def state(t):                          # (h, c) entering step t and h' leaving it (c: None for the tanh RNN)
            if not window:
                return b['rec_h'][t], b['rec_c'][t] if hc else None, b['rec_h'][t + 1]
            k, j = divmod(t, W)                # window mode: in the window buffers, entered from checkpoint k
            wh = b['win_h'][k % nb]
            if j == 0:
                return b['ck_h'][k], b['ck_c'][k] if hc else None, wh[0]
            return wh[j - 1], b['win_c'][k % nb][j - 1] if hc else None, wh[j]
        # window mode: window k, steps [t0, t1), is re-run on this stream right before ic3_bptt_step(t1 + 1) is issued
        # (before ic3_bptt_begin when there is no such step).  The look-ahead ic3_bptt_prepare(t) on the library's side
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
        _lib.check(lib.ic3_bptt_begin(C.byref(plan), cmax, s))
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
        FF_CHUNK_ROWS (at least one step)."""
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

    def _compute_grad_ff(self, adv, ret):
        """grad_impl 'kernels_ff' (ic3_ff_grad_*): the rollout's T lock-steps in chunks of K consecutive steps, each one
        batch of K*B env slots (records are [T, B, ...]), in any order since no state crosses a step; the backward's
        products run on the tensor cores.  Returns the device float64 vector of the three loss sums."""
        b, net, args, e = self._buf, self.policy_net, self.args, self.env.env
        lib = _lib.load()
        T, B, N = b['T'], e.nenvs, args.nagents
        s = _lib.stream()
        cfg = self._policy_cfg()
        w = net.packed()
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
        batch, stat = self.run_batch(epoch)
        if self.random_policy:
            # no gradient: the reference's step skips a parameter whose .grad is None (trainer.py:251-254), so the
            # parameter and the optimizer state (state == {}) stay as they are
            merge_stat(self.compute_grad(batch), stat)
            return stat
        self.optimizer.zero_grad(set_to_none=False)
        s = self.compute_grad(batch)
        merge_stat(s, stat)
        self.optimizer.step(grad_div=stat['num_steps'])      # grad /= num_steps, then the update (trainer.py:251-254)
        return stat

    def state_dict(self):
        return self.optimizer.state_dict()

    def load_state_dict(self, state):
        self.optimizer.load_state_dict(state)
