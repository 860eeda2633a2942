"""Evaluation recorder behind ``Trainer.evaluate_trace``: per-step trajectories of chosen evaluation slots and a map of
where agents open their communication gate, kept on the device while the evaluation plays (csrc/eval_trace.cu,
ic3_trace_step / ic3_comm_map_step) and copied to the host once at the end.  With ``messages`` it also keeps what the
agents send and receive (ic3_trace_comm_step / ic3_message_map_step), read before each policy step overwrites h.

Every array lives in one device byte arena, each behind a 16-byte guard band that no kernel writes, so the whole
recording comes back in one device->host copy."""
import ctypes as C

import numpy as np
import torch

from . import _lib

GUARD = 16
GUARD_BYTE = 0xA5


def parse_slots(slots, nenvs):
    """Local slot numbers of a slots argument: an int K (the first K slots) or a sequence of distinct slot numbers in
    [0, nenvs).  Raises ValueError otherwise."""
    if isinstance(slots, (int, np.integer)):
        k = int(slots)
        if not 1 <= k <= nenvs:
            raise ValueError("evaluate_trace records 1 .. %d slots, not %d" % (nenvs, k))
        return tuple(range(k))
    out = tuple(int(s) for s in slots)
    if not out:
        raise ValueError("evaluate_trace needs at least one slot")
    if len(set(out)) != len(out):
        raise ValueError("evaluate_trace slots must be distinct: %r" % (out,))
    bad = [s for s in out if not 0 <= s < nenvs]
    if bad:
        raise ValueError("evaluate_trace slots %r lie outside the %d evaluation slots" % (bad, nenvs))
    return out


class EvalTraceResult(object):
    """Trajectories of K evaluation slots over T = episodes * max_steps lock-steps (numpy, [T, K, ...]): loc and
    loc_next [T, K, rows, 2] int16 (entering step t; after its move, before the auto-reset), alive [T, K, NA] uint8,
    action [T, K, NA, nheads] int8, value and reward [T, K, NA] float32, t_ep [T, K] int16, done, success and valid
    [T, K] uint8, comm_prob [T, K, NA] float32 (with --hard_attn, else None), route_id [T, K, N] int16 (traffic junction,
    else None) and env_id [K] (global env ids).  With messages: msg_h and msg_in [T, K, NA, H] float32 (the hidden
    state each agent sends entering step t, and the communication vector S it receives) and msg_gate [T, K, NA] uint8
    (its gate g); else None."""
    FIELDS = ('loc', 'loc_next', 'alive', 'action', 'value', 'reward', 't_ep', 'done', 'success', 'valid', 'comm_prob',
              'route_id', 'env_id', 'msg_h', 'msg_gate', 'msg_in')

    def __init__(self, **arrays):
        for k in self.FIELDS:
            setattr(self, k, arrays.get(k))

    def arrays(self):
        """{field: array} of the fields this trace holds."""
        return {k: getattr(self, k) for k in self.FIELDS if getattr(self, k) is not None}


class Recorder(object):
    """The device buffers of one evaluate_trace configuration and the launches that fill them.  pre_step(t) runs before
    policy step t, step(t) between policy step t and env step t, finish(T) after the last env step; rollout_fields()
    are the ic3_rollout_io hooks the env step fills for it."""

    MSG_SCALE = 2.0 ** -32            # a message map sum times this is the sum of the float messages

    def __init__(self, trainer, e, b, T, slots, comm_map, messages=False):
        args = trainer.args
        dev = e.device
        self.e, self.b, self.T, self.K = e, b, int(T), len(slots)
        self.slots = slots
        self.is_tj = trainer.is_tj
        self.hard = trainer.hard
        NA = args.nagents
        rows = e.cfg.N if self.is_tj else e.cfg.N + 1
        heads = list(args.naction_heads)
        self.npos = e.cfg.h * e.cfg.w if self.is_tj else e.cfg.dim * e.cfg.dim
        self.max_steps = int(args.max_steps)
        T, K = self.T, self.K
        i16, u8 = torch.int16, torch.uint8
        spec = [('loc', (T, K, rows, 2), i16), ('loc_next', (T, K, rows, 2), i16), ('alive', (T, K, NA), u8),
                ('action', (T, K, NA, len(heads)), torch.int8), ('value', (T, K, NA), torch.float32),
                ('reward', (T, K, NA), torch.float32), ('t_ep', (T, K), i16), ('done', (T, K), u8),
                ('success', (T, K), u8), ('valid', (T, K), u8)]
        if self.hard:
            spec.append(('comm_prob', (T, K, NA), torch.float32))
        if self.is_tj:
            spec.append(('route_id', (T, K, NA), i16))
        self.messages = bool(messages)
        self.H = int(args.hid_size)
        if self.messages:
            spec += [('msg_h', (T, K, NA, self.H), torch.float32), ('msg_gate', (T, K, NA), u8),
                     ('msg_in', (T, K, NA, self.H), torch.float32)]
        self.map_keys = self._map_keys() if comm_map else []
        nmap = sum(n for _, n in self.map_keys)
        if nmap:
            spec.append(('counts', (nmap,), torch.int64))
        # message map (ic3_message_map_step): sent [R, H], recv [R, H], senders [R] over R key rows
        self.msg_rows = self.npos + self.max_steps + (0 if self.is_tj else 2)
        if self.messages and comm_map:
            spec.append(('msg_sums', ((2 * self.H + 1) * self.msg_rows,), torch.int64))
        spec += [('slots', (K,), torch.int32), ('out_loc', (e.nenvs, rows, 2), torch.int32),
                 ('out_success', (e.nenvs,), u8)]
        # arena: [guard][array][pad to 16][guard][array]...[guard]
        off, self.layout = GUARD, {}
        for name, shape, dt in spec:
            nbytes = int(np.prod(shape)) * torch.empty((), dtype=dt).element_size()
            self.layout[name] = (off, nbytes, shape, dt)
            off += (nbytes + 15) // 16 * 16 + GUARD
        self.arena = torch.full((off,), GUARD_BYTE, dtype=torch.uint8, device=dev)
        self.t = {name: self.arena[o:o + n].view(dt).view(shape) for name, (o, n, shape, dt) in self.layout.items()}
        self.t['slots'].copy_(torch.tensor(slots, dtype=torch.int32))
        self.t['out_loc'].zero_()
        self.t['out_success'].zero_()
        self.counts = self.t.get('counts')
        self.msg_sums = self.t.get('msg_sums')
        self.host_names = [n for n, _, _ in spec if n not in ('slots', 'out_loc', 'out_success')]
        pp = not self.is_tj
        self.io = _lib.EvalStepIO(
            pp_env=C.pointer(e.cfg) if pp else None, pp_state=C.pointer(e.state) if pp else None,
            tj_env=C.pointer(e.cfg) if not pp else None, tj_state=C.pointer(e.state) if not pp else None,
            nheads=len(heads), logp_cols=sum(heads), comm_col=sum(heads) - heads[-1] + 1 if self.hard else -1,
            max_steps=self.max_steps, t_ep=b['t_ep'].data_ptr(), halted=b['halted'].data_ptr(),
            action=b['action'][0].data_ptr(), value=b['value'][0].data_ptr(), logp=b['logp'][0].data_ptr(),
            reward=b['step_reward'].data_ptr(), fresh=b['fresh'].data_ptr(), out_loc=self.t['out_loc'].data_ptr(),
            out_success=self.t['out_success'].data_ptr(), err=b['err'].data_ptr())
        p = lambda k: self.t[k].data_ptr() if k in self.t else None
        self.tr = _lib.EvalTrace(T=T, K=K, slots=p('slots'), loc=p('loc'), loc_next=p('loc_next'), alive=p('alive'),
                                 action=p('action'), value=p('value'), reward=p('reward'), t_ep=p('t_ep'),
                                 done=p('done'), success=p('success'), valid=p('valid'), comm_prob=p('comm_prob'),
                                 route_id=p('route_id'))
        if self.messages:
            self.comm_io = _lib.EvalCommIO(h=b['h'].data_ptr(), comm=b['comm'].data_ptr() if self.hard else None,
                                           alive=b['alive'].data_ptr(), fresh=b['fresh'].data_ptr(), H=self.H,
                                           comm_avg=int(getattr(args, 'comm_mode', 'avg') == 'avg'),
                                           hard=int(self.hard))

    def _map_keys(self):
        """(key, length) of the comm-map blocks in ic3_comm_map_step's layout."""
        S, P = self.max_steps, self.npos
        keys = [('visits', P)] + ([('open', P)] if self.hard else []) + [('visits_t', S)] + \
            ([('open_t', S)] if self.hard else [])
        if not self.is_tj:
            keys += [('visits_reached', 2)] + ([('open_reached', 2)] if self.hard else [])
        return keys

    def rollout_fields(self):
        return dict(out_loc=self.t['out_loc'].data_ptr(), out_success=self.t['out_success'].data_ptr())

    def begin(self):
        if self.counts is not None:
            self.counts.zero_()
        if self.msg_sums is not None:
            self.msg_sums.zero_()

    def pre_step(self, t, s):
        """Before policy step t: the messages of step t, read from h before the step overwrites it."""
        if not self.messages:
            return
        lib = _lib.load()
        _lib.check(lib.ic3_trace_comm_step(C.byref(self.io), C.byref(self.comm_io), C.byref(self.tr),
                                           self.t['msg_h'].data_ptr(), self.t['msg_gate'].data_ptr(),
                                           self.t['msg_in'].data_ptr(), t, s))
        if self.msg_sums is not None:
            _lib.check(lib.ic3_message_map_step(C.byref(self.io), C.byref(self.comm_io), self.msg_sums.data_ptr(), s))

    def step(self, t, s):
        lib = _lib.load()
        _lib.check(lib.ic3_trace_step(C.byref(self.io), C.byref(self.tr), t, s))
        if self.counts is not None:
            _lib.check(lib.ic3_comm_map_step(C.byref(self.io), self.counts.data_ptr(), s))

    def finish(self, T, s):
        _lib.check(_lib.load().ic3_trace_step(C.byref(self.io), C.byref(self.tr), T, s))

    def guards_intact(self):
        """Every guard band of the arena still holds its fill byte (no kernel wrote past an array)."""
        a = self.arena.cpu().numpy()
        ends = sorted((o, o + (n + 15) // 16 * 16) for o, n, _, _ in self.layout.values())
        spans = [(0, GUARD)] + [(end, end + GUARD) for _, end in ends]
        return all((a[lo:hi] == GUARD_BYTE).all() for lo, hi in spans) and \
            all((a[o + n:o + (n + 15) // 16 * 16] == GUARD_BYTE).all() for o, n, _, _ in self.layout.values())

    def to_host(self):
        """(EvalTraceResult, comm map dict or None) from one device->host copy of the arena."""
        host = self.arena.cpu().numpy()
        npdt = {torch.int16: np.int16, torch.uint8: np.uint8, torch.int8: np.int8, torch.float32: np.float32,
                torch.int64: np.int64, torch.int32: np.int32}
        get = lambda name: host[self.layout[name][0]:self.layout[name][0] + self.layout[name][1]].view(
            npdt[self.layout[name][3]]).reshape(self.layout[name][2]).copy()
        arrays = {n: get(n) for n in self.host_names if n not in ('counts', 'msg_sums')}
        arrays['env_id'] = int(self.e.cfg.env_id0) + np.asarray(self.slots, dtype=np.int64)
        cmap = None
        if self.counts is not None:
            c = get('counts')
            cmap, o = {}, 0
            for key, n in self.map_keys:
                cmap[key] = c[o:o + n].copy()
                o += n
        if self.msg_sums is not None:
            cmap.update(self._message_map(get('msg_sums'), cmap))
        return EvalTraceResult(**arrays), cmap

    def _message_map(self, sums, cmap):
        """The message map's blocks under msg_* keys: int64 sums of sent and received messages (scale msg_scale) by
        cell, by episode step and, predator-prey, on / off the prey; the open senders' counts; and float64 means
        where a count exists (NaN elsewhere): sent over the open senders, received over every counted agent (the comm
        map's visits)."""
        R, H, P, S = self.msg_rows, self.H, self.npos, self.max_steps
        sent, recv, senders = sums[:R * H].reshape(R, H), sums[R * H:2 * R * H].reshape(R, H), sums[2 * R * H:]
        parts = [('', slice(0, P), 'visits'), ('_t', slice(P, P + S), 'visits_t')]
        if not self.is_tj:
            parts.append(('_reached', slice(P + S, R), 'visits_reached'))
        out = dict(msg_scale=np.float64(self.MSG_SCALE))

        def mean(total, n):
            n = n.astype(np.float64)[:, None]
            with np.errstate(invalid='ignore', divide='ignore'):
                return np.where(n > 0, total.astype(np.float64) * self.MSG_SCALE / n, np.nan)
        for suffix, rows, visits in parts:
            out['msg_sent' + suffix] = sent[rows].copy()
            out['msg_recv' + suffix] = recv[rows].copy()
            out['msg_senders' + suffix] = senders[rows].copy()
            out['msg_sent_mean' + suffix] = mean(sent[rows], senders[rows])
            out['msg_recv_mean' + suffix] = mean(recv[rows], cmap[visits])
        return out
