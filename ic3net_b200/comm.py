"""CommNet / IC3Net policy on one GPU, behind the reference's ``comm.CommNetMLP``
surface (comm.py:8-253): ``CommNetMLP(args, num_inputs)``, ``forward(x, info={})``,
``init_hidden(batch_size)`` and the same ``state_dict`` keys
(``heads.k.*``, ``encoder.*``, ``hidd_encoder.*``, ``f_module.{weight,bias}_{ih,hh}``,
``C_modules.0.*``, ``value_head.*``), so checkpoints interchange.

The forward pass runs the hand-written kernels of csrc/policy.cu through the C ABI
(encoder, gated hidden-state mean, C, LSTMCell, value/action heads) in float32 for a
whole batch ``[B, N, .]`` of environments.  The recurrent (LSTM) branch with one comm pass -- the
branch every BASELINE config uses -- runs on the wgmma tensor-core kernels; ``comm_passes > 1``,
``share_weights`` and the non-recurrent tanh branch (comm.py:63-70,127-131,220-224) run on the
fp32 SIMT kernel.  By default ``forward`` is inference-only (the reference detaches what it samples from,
action_utils.py:35) and gradients are taken by the trainer.  With ``args.forward_grad = 'kernels'`` its outputs carry
a ``grad_fn`` whenever grad mode is on and a parameter requires grad: the backward of the step runs on the hand-written
BPTT kernels (ic3_policy_step_backward, csrc/bptt_tc.cu), so a driver can differentiate its own loss through the
module as the reference's Trainer does (trainer.py:54-60,223).  It covers what those kernels cover at hid_size 128 --
the LSTM CommNet / IC3Net on policy_impl 'tc' (1..4 comm passes, share_weights), models.RNN with the LSTM cell, and the
tanh RNN of the IC / IRIC baselines -- on observation handles (LazyObs, args.obs_api = 'handle').
"""
import ctypes as C
import weakref

import numpy as np
import torch
from torch import nn
from torch.autograd.function import once_differentiable

from . import _lib
from .lazy_obs import LazyObs


def _as_u8(v, B, N, device):
    """info['comm_action'] / info['alive_mask'] (numpy or tensor, [N] or [B,N]) -> uint8 [B,N]."""
    if torch.is_tensor(v) and v.dtype == torch.uint8 and tuple(v.shape) == (B, N) and v.is_contiguous():
        return v if v.is_cuda else v.to(device, non_blocking=True)     # the common case: one (async if pinned) copy
    if torch.is_tensor(v) and v.is_cuda:
        t = v if v.dtype == torch.uint8 else (v != 0).to(torch.uint8)
    else:       # host mask: normalise on the host, then ONE copy (asynchronous when the source is pinned)
        t = v if torch.is_tensor(v) else torch.from_numpy(np.ascontiguousarray(np.asarray(v)))
        if t.dtype != torch.uint8:
            t = (t != 0).to(torch.uint8)
        t = t.to(device, non_blocking=True)
    if t.dim() == 1:
        t = t.unsqueeze(0).expand(B, N)
    return t.reshape(B, N).contiguous()      # the kernels test `!= 0`, any non-zero byte counts as 1


class CommNetMLP(nn.Module):
    # kernel-side description of the variant (include/ic3net_b200.h, ic3_policy_cfg.cell / passes / x_tanh / h_from_x)
    def _variant(self, args):
        rec = bool(args.recurrent)
        return dict(cell=_lib.CELL_LSTM if rec else _lib.CELL_TANH, passes=int(args.comm_passes),
                    x_tanh=0 if rec else 1, h_from_x=0 if rec else 1)

    def _build_modules(self, args, num_inputs):
        """Parameters with the reference's names and shapes (comm.py:31-96); init like nn.Linear / nn.LSTMCell."""
        H = args.hid_size
        self.heads = nn.ModuleList([nn.Linear(H, o) for o in args.naction_heads])
        self.encoder = nn.Linear(num_inputs, H)
        if args.recurrent:
            self.hidd_encoder = nn.Linear(H, H)          # allocated but unused by the reference forward (comm.py:57,125)
            self.f_module = nn.LSTMCell(H, H)
        elif args.share_weights:                          # comm.py:63-66: one module repeated in the list
            self.f_module = nn.Linear(H, H)
            self.f_modules = nn.ModuleList([self.f_module for _ in range(self.comm_passes)])
        else:
            self.f_modules = nn.ModuleList([nn.Linear(H, H) for _ in range(self.comm_passes)])
        if args.share_weights:                            # comm.py:76-79
            self.C_module = nn.Linear(H, H)
            self.C_modules = nn.ModuleList([self.C_module for _ in range(self.comm_passes)])
        else:
            self.C_modules = nn.ModuleList([nn.Linear(H, H) for _ in range(self.comm_passes)])
        if args.comm_init == 'zeros':                     # comm.py:86-88
            for i in range(self.comm_passes):
                self.C_modules[i].weight.data.zero_()
        self.value_head = nn.Linear(H, 1)

    def _kernel_weights(self):
        """The tensors the kernels consume, by role (subclasses in models.py map their own parameter names here)."""
        w = dict(enc_w=self.encoder.weight, enc_b=self.encoder.bias,
                 c_w=[m.weight for m in self.C_modules], c_b=[m.bias for m in self.C_modules],
                 value_w=self.value_head.weight, value_b=self.value_head.bias,
                 head_w=[h.weight for h in self.heads], head_b=[h.bias for h in self.heads])
        if self.recurrent:
            w.update(w_ih=self.f_module.weight_ih, w_hh=self.f_module.weight_hh, b_ih=self.f_module.bias_ih,
                     b_hh=self.f_module.bias_hh)
        else:
            w.update(f_w=[m.weight for m in self.f_modules], f_b=[m.bias for m in self.f_modules])
        return w

    def __init__(self, args, num_inputs):
        super(CommNetMLP, self).__init__()
        _lib.require_cuda()
        self.args = args
        self.nagents = args.nagents
        self.hid_size = args.hid_size
        self.comm_passes = args.comm_passes
        self.recurrent = args.recurrent
        self.continuous = args.continuous
        if self.continuous:
            raise NotImplementedError("continuous actions are outside the accelerated path")
        if args.recurrent and getattr(args, 'rnn_type', 'LSTM') != 'LSTM':
            raise NotImplementedError("recurrent CommNet needs rnn_type LSTM (main.py:151-153 forces it)")
        if not 1 <= int(args.comm_passes) <= _lib.MAX_PASSES:
            raise NotImplementedError("comm_passes must be in 1..%d" % _lib.MAX_PASSES)
        self.num_inputs = num_inputs
        H = args.hid_size
        self._build_modules(args, num_inputs)
        self._dev = torch.device('cuda', torch.cuda.current_device())
        self.to(self._dev, torch.float32)

        heads = list(args.naction_heads)
        self._atot = sum(heads)
        hd = (C.c_int32 * _lib.MAX_HEADS)(*(heads + [0] * (_lib.MAX_HEADS - len(heads))))
        var = self._variant(args)
        self.is_variant = (var['cell'] != _lib.CELL_LSTM or var['passes'] > 1 or var['x_tanh'] or var['h_from_x'])
        self._cfg_proto = dict(N=self.nagents, H=H, O=num_inputs, nheads=len(heads), head_dim=hd,
                               hard_attn=int(bool(args.hard_attn)),
                               comm_avg=int(getattr(args, 'comm_mode', 'avg') == 'avg'),
                               comm_mask_zero=int(bool(args.comm_mask_zero)),
                               env_id0=int(getattr(args, 'env_id0', 0)),
                               seed=int(getattr(args, 'seed', 0)) & 0xFFFFFFFFFFFFFFFF,
                               obs_off=0, obs_vocab=0, obs_ncount=0, **var)
        self._plist = None
        self._packed = None
        self._packed_key = None
        # 'tc' = wgmma tensor-core path (csrc/policy_tc.cu: hid_size 128, LSTM cell on the encoded observation, any
        # number of comm passes), 'simt' = fp32 CUDA-core kernel (every variant), 'tc_tanh' = wgmma step of the tanh RNN
        # without communication (csrc/ff_tc.cu: models.RNN with the vanilla recurrence, hid_size 128); opt-in;
        # 'tc_ff' = wgmma step of the non-recurrent tanh policies (csrc/ff_tc.cu: models.MLP, CommNet / IC3Net without
        # --recurrent, hid_size 128); opt-in
        self.tc_capable = (var['cell'] == _lib.CELL_LSTM and not var['x_tanh'] and not var['h_from_x'])
        want = getattr(args, 'policy_impl', None)
        self.policy_impl = want or ('tc' if (H == 128 and self.tc_capable) else 'simt')
        if self.policy_impl not in ('tc', 'simt', 'tc_tanh', 'tc_ff'):
            raise ValueError("policy_impl must be 'tc', 'simt', 'tc_tanh' or 'tc_ff'")
        if self.policy_impl != 'simt' and H != 128:
            raise NotImplementedError("the tensor-core policy path is specialised for hid_size 128")
        if self.policy_impl == 'tc_ff' and not (var['cell'] == _lib.CELL_TANH and var['x_tanh'] and var['h_from_x']):
            raise NotImplementedError("policy_impl='tc_ff' implements the non-recurrent tanh step (models.MLP, CommNet / "
                                      "IC3Net without --recurrent); recurrent LSTM cells run on 'tc', the tanh RNN "
                                      "(IC / IRIC) on 'tc_tanh'")
        if self.policy_impl == 'tc_tanh' and not (var['cell'] == _lib.CELL_TANH and var['passes'] == 1 and
                                                  args.comm_mask_zero and not args.hard_attn and
                                                  not var['x_tanh'] and not var['h_from_x']):
            raise NotImplementedError("policy_impl='tc_tanh' implements the tanh RNN without communication (models.RNN "
                                      "with rnn_type 'MLP': the IC / IRIC baselines); LSTM cells run on 'tc', models.MLP "
                                      "and the non-recurrent CommNet / IC3Net on 'simt'")
        if self.policy_impl == 'tc' and not self.tc_capable:
            raise NotImplementedError("the tensor-core policy path implements the recurrent LSTM policy; the tanh-cell "
                                      "variants run on policy_impl='simt'")
        self._ws = {}
        self._enc_tables = weakref.WeakKeyDictionary()     # env -> (packed-weights key, encoder_table(env))
        # differentiable forward on the BPTT kernels (ic3_policy_step_backward); None = inference-only forward
        self.forward_grad = getattr(args, 'forward_grad', None)
        if self.forward_grad not in (None, 'kernels'):
            raise ValueError("forward_grad must be None or 'kernels'")
        if self.forward_grad:
            lstm_tc = var['cell'] == _lib.CELL_LSTM and self.policy_impl == 'tc'
            tanh_rnn = (var['cell'] == _lib.CELL_TANH and not var['x_tanh'] and not var['h_from_x'] and
                        var['passes'] == 1 and args.comm_mask_zero and not args.hard_attn and
                        self.policy_impl in ('simt', 'tc_tanh'))
            if H != 128 or not (lstm_tc or tanh_rnn):
                raise NotImplementedError("forward_grad='kernels' covers the recurrent LSTM CommNet / IC3Net on "
                                          "policy_impl='tc' (1..%d comm passes), models.RNN and the tanh RNN of the IC / "
                                          "IRIC baselines, at hid_size 128; models.MLP and the non-recurrent CommNet / "
                                          "IC3Net have no differentiable forward" % _lib.MAX_PASSES)
        self._bwd_ws = {}                                   # B -> workspace of ic3_policy_step_backward

    def set_obs_layout(self, off, vocab, ncount):
        """Observation layout hint (include/ic3net_b200.h, ic3_policy_cfg.obs_vocab): lets the encoder sum the
        one-hot class terms separately from the counts, so the class part can come from a per-position table and
        the dense / index / fused encoders stay bit-identical.  (0, 0, 0) = plain single sum."""
        self._cfg_proto.update(obs_off=int(off), obs_vocab=int(vocab), obs_ncount=int(ncount))

    def fuses_encoder(self, env):
        """Whether the policy step can form x from the env state itself (the fused index encoder): the tensor-core
        path, with a vision window of at most 5x5, on the traffic junction's bool vocabulary only (a scalar-vocabulary
        env's x comes from the separate index / dense encoder)."""
        W = 2 * env.vision + 1
        return self.policy_impl == 'tc' and W * W <= 25 and getattr(env, 'vocab_type', 'bool') == 'bool'

    def encoder_table(self, env, force=False):
        """[positions, H] class part of x per agent position of env (ic3_*_encoder_table) for the current packed
        weights, rebuilt when they change (force: always, for a CUDA graph that replays the build); one table per
        environment.  None where the fused index encoder takes no table: no fused encoder (fuses_encoder), or a layout
        without separate class terms (obs_vocab = 0)."""
        if not self.fuses_encoder(env) or self._cfg_proto['obs_vocab'] == 0:
            return None
        w = self.packed()
        key, table = self._enc_tables.get(env, (None, None))
        if table is None:
            table = torch.empty(env.obs_positions, self.hid_size, device=self._dev)
        if force or key != self._packed_key:
            lib = _lib.load()
            fn = lib.ic3_tj_encoder_table if isinstance(env.cfg, _lib.TJCfg) else lib.ic3_pp_encoder_table
            cfg = self.policy_cfg(env.nenvs)
            _lib.check(fn(C.byref(env.cfg), C.byref(cfg), C.byref(w), table.data_ptr(), _lib.stream()))
            self._enc_tables[env] = (self._packed_key, table)
        return table

    # ---- kernel-side weights ---------------------------------------------------
    def policy_cfg(self, B):
        return _lib.PolicyCfg(B=B, **self._cfg_proto)

    def workspace(self, B):
        """(scratch, err) tensors of the tensor-core paths for a batch of B envs (None, None for 'simt')."""
        if self.policy_impl == 'simt':
            return None, None
        if B not in self._ws:
            cfg = self.policy_cfg(B)
            nbytes = int(_lib.load().ic3_policy_workspace_bytes(C.byref(cfg)))
            dev = self._dev
            self._ws[B] = (torch.empty(nbytes, dtype=torch.uint8, device=dev),
                           torch.zeros(1, dtype=torch.int32, device=dev))
        return self._ws[B]

    def _param_list(self):
        """Flat list of the kernel-side tensors.  Cached: the Parameter OBJECTS of a module stay the same through
        load_state_dict / optimizer steps / re-pointed ``.data`` (all seen by packed()'s data_ptr + version key);
        ``_apply`` (``.to`` / ``.cuda`` / ``.float``) drops the cache, and code that assigns a NEW Parameter object
        to a submodule calls ``invalidate_packed()``."""
        if self._plist is None:
            ps = []
            for v in self._kernel_weights().values():
                ps += list(v) if isinstance(v, (list, tuple)) else [v]
            self._plist = ps
        return self._plist

    def invalidate_packed(self):
        self._plist = None
        self._packed_key = None

    def _apply(self, fn, *a, **kw):
        self.__dict__['_plist'] = None
        return super(CommNetMLP, self)._apply(fn, *a, **kw)

    def load_state_dict(self, *a, **kw):
        out = super(CommNetMLP, self).load_state_dict(*a, **kw)
        self.invalidate_packed()             # assign=True installs new Parameter objects
        return out

    def packed(self, force=False):
        """K-major kernel layout of the parameters; re-packed (one kernel) when any parameter changed, or always with
        force (a CUDA graph capturing the pack, Trainer graph_update)."""
        ps = self._param_list()
        key = tuple((p.data_ptr(), p._version) for p in ps)
        if self._packed is not None and key == self._packed_key and not force:
            return self._packed
        H, O, P = self.hid_size, self.num_inputs, self.comm_passes
        dev = ps[0].device
        w = self._kernel_weights()
        lstm = 'w_ih' in w
        if self._packed is None:
            nout = 1 + self._atot
            self._bufs = dict(enc_wT=torch.empty(O, H, device=dev), enc_b=torch.empty(H, device=dev),
                              c_wT=torch.empty(P, H, H, device=dev), c_b=torch.empty(P, H, device=dev),
                              lstm_wT=torch.empty(2 * H, 4 * H, device=dev), lstm_b=torch.empty(4 * H, device=dev),
                              head_w=torch.empty(nout, H, device=dev), head_b=torch.empty(nout, device=dev))
            if not lstm:
                self._bufs['f_wT'] = torch.empty(P, H, H, device=dev)
                self._bufs['f_b'] = torch.empty(P, H, device=dev)
            if self.policy_impl == 'tc':
                self._bufs['lstm_img'] = torch.empty(P * _lib.LSTM_IMG_BYTES, dtype=torch.uint8, device=dev)   # one per pass
                self._bufs['bias_cat'] = torch.empty(P, 4 * H, device=dev)
                self._bufs['flags'] = torch.zeros(1, dtype=torch.int32, device=dev)
            if self.policy_impl in ('tc_tanh', 'tc_ff'):     # one F (and C) image per pass
                nbytes = _lib.ff_img_bytes(P, not self._cfg_proto['comm_mask_zero'])
                self._bufs['ff_img'] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
                self._bufs['flags'] = torch.zeros(1, dtype=torch.int32, device=dev)
            self._packed = _lib.PolicyPacked(**{k: v.data_ptr() for k, v in self._bufs.items()})
        for p in ps:
            assert p.is_cuda and p.dtype == torch.float32 and p.is_contiguous()
        nh = len(w['head_w'])
        arr = lambda lst, n: (C.c_void_p * n)(*([t.data_ptr() for t in lst] + [None] * (n - len(lst))))
        kw = dict(encoder_w=w['enc_w'].data_ptr(), encoder_b=w['enc_b'].data_ptr(), c_w=w['c_w'][0].data_ptr(),
                  c_b=w['c_b'][0].data_ptr(), value_w=w['value_w'].data_ptr(), value_b=w['value_b'].data_ptr(),
                  head_w=arr(w['head_w'], _lib.MAX_HEADS), head_b=arr(w['head_b'], _lib.MAX_HEADS),
                  c_w_pass=arr(w['c_w'], _lib.MAX_PASSES), c_b_pass=arr(w['c_b'], _lib.MAX_PASSES))
        if lstm:
            kw.update(w_ih=w['w_ih'].data_ptr(), w_hh=w['w_hh'].data_ptr(), b_ih=w['b_ih'].data_ptr(),
                      b_hh=w['b_hh'].data_ptr())
        else:
            kw.update(f_w_pass=arr(w['f_w'], _lib.MAX_PASSES), f_b_pass=arr(w['f_b'], _lib.MAX_PASSES))
        params = _lib.PolicyParams(**kw)
        cfg = self.policy_cfg(1)
        _lib.check(_lib.load().ic3_policy_pack(C.byref(cfg), C.byref(params), C.byref(self._packed), _lib.stream()))
        self._packed_key = key
        return self._packed

    def mark_packed_current(self, envs=()):
        """A replayed CUDA graph has just re-packed the current parameters and re-built the encoder tables of envs: take
        the parameters' present version counters as the key of those, so packed() and encoder_table() keep them."""
        key = tuple((p.data_ptr(), p._version) for p in self._param_list())
        for env in envs:
            if env in self._enc_tables:          # none where the layout has no separate class terms (encoder_table)
                self._enc_tables[env] = (key, self._enc_tables[env][1])
        self._packed_key = key

    def policy_params(self, get):
        """ic3_policy_params with get(tensor) for every kernel-side tensor by role: get = data_ptr gives the parameters,
        a map to gradient buffers gives the gradient struct of ic3_bptt_finish / ic3_policy_step_backward."""
        w = self._kernel_weights()
        arr = lambda lst: (C.c_void_p * _lib.MAX_HEADS)(*([get(t) for t in lst] + [None] * (_lib.MAX_HEADS - len(lst))))
        # C_modules[p] per comm pass (share_weights: the same module, so the gradient pointers alias)
        parr = lambda lst: (C.c_void_p * _lib.MAX_PASSES)(*([get(t) for t in lst] + [None] * (_lib.MAX_PASSES - len(lst))))
        # the LSTM cell's w_ih / w_hh / b_ih / b_hh, or the tanh cell's f_w / f_b per pass
        cell = (dict(w_ih=get(w['w_ih']), w_hh=get(w['w_hh']), b_ih=get(w['b_ih']), b_hh=get(w['b_hh']))
                if 'w_ih' in w else dict(f_w_pass=parr(w['f_w']), f_b_pass=parr(w['f_b'])))
        return _lib.PolicyParams(encoder_w=get(w['enc_w']), encoder_b=get(w['enc_b']), c_w=get(w['c_w'][0]),
                                 c_b=get(w['c_b'][0]), value_w=get(w['value_w']), value_b=get(w['value_b']),
                                 head_w=arr(w['head_w']), head_b=arr(w['head_b']),
                                 c_w_pass=parr(w['c_w']), c_b_pass=parr(w['c_b']), **cell)

    def check_errors(self):
        """Raise if a forward() of this module set a device-side error flag (tensor-core path: pipeline watchdog, fp16
        operand range).  One host synchronisation; the trainer checks its own flag word in collect_stat."""
        for ws, err in self._ws.values():
            flags = int(err.item())
            if flags:
                raise RuntimeError("device-side error flag %#x in CommNetMLP.forward" % flags)

    # ---- reference surface -------------------------------------------------------
    def forward(self, x, info={}):
        """Recurrent: x = [state [B,N,O], (h, c) each [B*N, H]] -> (list of log-probs [B,N,na_k], value [B*N,1],
        (h', c')); non-recurrent: x = state -> (log-probs, value)  (comm.py:134-244).  info may hold 'comm_action' and
        'alive_mask' ([N] or [B,N])."""
        lstm = self._cfg_proto['cell'] == _lib.CELL_LSTM
        carries = not self._cfg_proto['h_from_x']               # a hidden state enters from the previous step
        if carries:
            state, hid = x
            h, c = hid if lstm else (hid, None)
        else:
            state, h, c = x, None, None
        B = state.shape[0]
        if self.forward_grad and torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            if not isinstance(state, LazyObs):
                raise NotImplementedError("forward_grad='kernels' differentiates observation handles only (LazyObs: "
                                          "args.obs_api='handle'); the backward rebuilds the observation from the env "
                                          "state")
            h = h.to(self._dev, torch.float32).reshape(B * self.nagents, self.hid_size)
            c = c.to(self._dev, torch.float32) if c is not None else None
            params = self._grad_params()
            out = _PolicyStep.apply(self, state, info, h, c, *params)
            action = list(torch.split(out[0], list(self.args.naction_heads), dim=-1))
            return action, out[1], ((out[2], out[3]) if lstm else out[2])
        logp, value, h2, c2, _ = self._step(state, h, c, info)
        action = list(torch.split(logp, list(self.args.naction_heads), dim=-1))
        if not carries:
            return action, value.view(B, self.nagents, 1)          # comm.py:243-244
        return action, value, ((h2, c2) if lstm else h2)

    def _step(self, state, h, c, info):
        """One ic3_policy_step on detached inputs: (log-probs [B, N, sum(na)], value [B*N, 1], h', c' or None, and the
        (policy cfg, comm_action, alive_mask) the kernel read)."""
        lstm = self._cfg_proto['cell'] == _lib.CELL_LSTM
        B, N, H = state.shape[0], self.nagents, self.hid_size
        dev = state.device
        lazy = isinstance(state, LazyObs)            # observation handle (lazy_obs.py): encoder from the env state
        if not lazy:
            state = state.to(torch.float32).contiguous()
        if h is not None:
            h = h.detach().to(dev, torch.float32).reshape(B * N, H).contiguous()
        if c is not None:
            c = c.detach().to(dev, torch.float32).contiguous()
        lib = _lib.load()
        src, xenc = {}, None
        if lazy:
            cfg, w, src, xenc = self._index_encoder(state, B)
        else:
            cfg = self.policy_cfg(B)
            w = self.packed()
            xenc = torch.empty(B * N, H, device=dev)
            _lib.check(lib.ic3_encoder_dense(C.byref(cfg), C.byref(w), state.data_ptr(), xenc.data_ptr(), _lib.stream()))
        comm = alive = None
        if self.args.hard_attn:
            comm = _as_u8(info['comm_action'], B, N, dev)          # comm.py:171-175
        if 'alive_mask' in info:
            alive = _as_u8(info['alive_mask'], B, N, dev)          # comm.py:102-104
        h2 = torch.empty(B * N, H, device=dev)
        c2 = torch.empty(B * N, H, device=dev) if lstm else None
        value = torch.empty(B * N, 1, device=dev)
        logp = torch.empty(B, N, self._atot, device=dev)
        ws, err = self.workspace(B)
        io = _lib.PolicyIO(x=_lib.ptr(xenc), h=_lib.ptr(h), c=_lib.ptr(c), comm_action=_lib.ptr(comm),
                           alive=_lib.ptr(alive), fresh=None, tick=None, draws=None, h_out=h2.data_ptr(),
                           c_out=_lib.ptr(c2), value=value.data_ptr(), logp=logp.data_ptr(), action=None,
                           workspace=_lib.ptr(ws), err=_lib.ptr(err), **src)
        _lib.check(lib.ic3_policy_step(C.byref(cfg), C.byref(w), C.byref(io), _lib.stream()))
        return logp, value, h2, c2, (cfg, comm, alive)

    def _grad_params(self):
        """The distinct Parameters among the kernel-side tensors (share_weights aliases once; frozen buffers left out):
        the inputs through which autograd hands ic3_policy_step_backward's gradients to them."""
        seen, out = set(), []
        for p in self._param_list():
            if isinstance(p, nn.Parameter) and id(p) not in seen:
                seen.add(id(p))
                out.append(p)
        return out

    def _bwd_plan(self, env, cfg, w):
        """ic3_bptt_plan of a differentiable step on env (the workspace is set by the backward); NotImplementedError
        where the BPTT kernels do not cover the policy on this environment."""
        table = self.encoder_table(env) if self._cfg_proto['cell'] == _lib.CELL_LSTM else None
        tj = isinstance(env.cfg, _lib.TJCfg)
        ecfg = type(env.cfg).from_buffer_copy(env.cfg)
        plan = _lib.BpttPlan(cfg=C.pointer(cfg), w=C.pointer(w), pp_env=None if tj else C.pointer(ecfg),
                             tj_env=C.pointer(ecfg) if tj else None, x_table=_lib.ptr(table), value_coeff=0.0,
                             entr=0.0, workspace=None)
        nbytes = int(_lib.load().ic3_bptt_workspace_bytes(C.byref(plan)))
        if nbytes == 0 or (self._cfg_proto['cell'] == _lib.CELL_LSTM and table is None):
            raise NotImplementedError("forward_grad='kernels' does not cover this environment: the BPTT kernels need a "
                                      "vision window of at most 5 x 5 cells, the traffic junction's bool vocabulary and "
                                      "at most 7 action logits")
        return plan, nbytes, (ecfg, table)

    def _index_encoder(self, obs, B):
        """Encoder input for an observation HANDLE: returns (cfg, packed weights, PolicyIO source fields, x tensor or
        None).  Where the policy has an encoder table for the env (encoder_table): the encoder is fused into the policy
        step (x is formed from the env state and the table inside the operand-preparation kernel); otherwise the
        index-form encoder kernel writes x.  Either way the same sums in the same order as ic3_encoder_dense."""
        e = obs.check_current()
        lib = _lib.load()
        if self._cfg_proto['obs_vocab'] == 0 and getattr(e, 'obs_layout', (0, 0, 0))[1]:
            self.set_obs_layout(*e.obs_layout)
        cfg = self.policy_cfg(B)
        cfg.seed, cfg.env_id0 = e.cfg.seed, e.cfg.env_id0
        w = self.packed()
        table = self.encoder_table(e)
        if table is not None:
            return cfg, w, dict(_lib.env_source(e.cfg, e.state), x_table=table.data_ptr()), None
        xenc = torch.empty(B * self.nagents, self.hid_size, device=self._dev)
        fn = lib.ic3_tj_encoder_index if isinstance(e.cfg, _lib.TJCfg) else lib.ic3_pp_encoder_index
        _lib.check(fn(C.byref(e.cfg), C.byref(e.state), C.byref(cfg), C.byref(w), xenc.data_ptr(), _lib.stream()))
        return cfg, w, {}, xenc

    def init_hidden(self, batch_size):
        dev = self._dev
        return tuple((torch.zeros(batch_size * self.nagents, self.hid_size, device=dev),
                      torch.zeros(batch_size * self.nagents, self.hid_size, device=dev)))


# env state fields the backward reads (ic3_policy_bwd_io.pp_state / tj_state): env attribute -> ic3_*_state field
_PP_BWD_STATE = (('loc', 'loc'),)
_TJ_BWD_STATE = (('car_loc', 'loc'), ('alive_mask', 'alive'), ('car_last_act', 'last_act'), ('route_id', 'route_id'))


class _PolicyStep(torch.autograd.Function):
    """CommNetMLP.forward with forward_grad='kernels': the module's own policy step forward (outputs bit-identical to
    the inference-only forward), ic3_policy_step_backward backward.  Saves the step's inputs and outputs and a copy of
    the env-state fields the backward reads (an observation handle is only valid until its env's next step); the packed
    weights and encoder table are the module's, checked unchanged through the parameters' data_ptr / _version."""

    @staticmethod
    def forward(ctx, net, obs, info, h, c, *params):
        logp, value, h2, c2, (cfg, comm, alive) = net._step(obs, h, c, info)
        env = obs.env
        w = net.packed()
        ctx.plan, ctx.nbytes, ctx.keep = net._bwd_plan(env, cfg, w)
        ctx.cfg, ctx.w, ctx.env = cfg, w, env
        ctx.key = net._packed_key
        tj = isinstance(env.cfg, _lib.TJCfg)
        copies = {field: getattr(env, attr).clone() for attr, field in (_TJ_BWD_STATE if tj else _PP_BWD_STATE)}
        ctx.state = (_lib.TJState if tj else _lib.PPState)(**{f: t.data_ptr() for f, t in copies.items()})
        ctx.tj = tj
        ctx.copies = copies
        ctx.comm = None if comm is None else comm.clone()
        ctx.alive = None if alive is None else alive.clone()
        ctx.net, ctx.nparams = net, len(params)
        ctx.set_materialize_grads(False)
        outs = (logp, value, h2) + ((c2,) if c2 is not None else ())
        ctx.save_for_backward(h, c, h2, logp)
        return outs

    @staticmethod
    @once_differentiable
    def backward(ctx, dlogp, dvalue, dh2, *rest):
        net = ctx.net
        if tuple((p.data_ptr(), p._version) for p in net._param_list()) != ctx.key:
            raise RuntimeError("a parameter of the policy was modified in place (e.g. by an optimizer step) between "
                               "this forward and its backward; the backward needs the weights of the forward")
        h, c, h2, logp = ctx.saved_tensors
        dc2 = rest[0] if rest else None
        R, H = h2.shape
        dev = h2.device
        ws = net._bwd_ws.get(R)
        if ws is None or ws.numel() < ctx.nbytes:
            ws = torch.empty(ctx.nbytes, dtype=torch.uint8, device=dev)
            net._bwd_ws[R] = ws
        plan = ctx.plan
        plan.workspace = ws.data_ptr()
        lstm = c is not None
        dh = torch.empty(R, H, device=dev)
        dc = torch.empty(R, H, device=dev) if lstm else None
        params = net._grad_params()
        grads = {id(p): torch.zeros_like(p) for p in params}
        scratch = {}                     # frozen kernel-side buffers (models.py zero comm projection): discarded

        def grad_ptr(t):
            g = grads.get(id(t))
            if g is None:
                g = scratch.setdefault(id(t), torch.zeros_like(t))
            return g.data_ptr()
        prm, grd = net.policy_params(lambda t: t.data_ptr()), net.policy_params(grad_ptr)
        # every tensor the call reads stays referenced here until it has been enqueued
        cont = lambda t: None if t is None else t.to(torch.float32).contiguous()
        h, c, dlogp, dvalue, dh2, dc2 = cont(h), cont(c), cont(dlogp), cont(dvalue), cont(dh2), cont(dc2)
        st = C.pointer(ctx.state)
        _, err = net.workspace(R // net.nagents)
        io = _lib.PolicyBwdIO(h_prev=h.data_ptr(), c_prev=_lib.ptr(c), h_new=h2.data_ptr(),
                              logp=logp.data_ptr(), comm=_lib.ptr(ctx.comm), alive=_lib.ptr(ctx.alive),
                              tj_state=st if ctx.tj else None, pp_state=None if ctx.tj else st,
                              dlogp=_lib.ptr(dlogp), dvalue=_lib.ptr(dvalue), dh_new=_lib.ptr(dh2), dc_new=_lib.ptr(dc2),
                              dh_prev=dh.data_ptr(), dc_prev=_lib.ptr(dc), err=_lib.ptr(err))
        _lib.check(_lib.load().ic3_policy_step_backward(C.byref(plan), C.byref(io), C.byref(prm), C.byref(grd),
                                                        _lib.stream()))
        return (None, None, None, dh, dc) + tuple(grads[id(p)] for p in params)
