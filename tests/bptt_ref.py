"""Float64 reference of the hand-written BPTT (csrc/bptt_tc.cu) on the kernel trainer's own records.

``trainer_reference(tr)`` differentiates the batch a ``Trainer`` with ``grad_kernels`` recorded in its last rollout:
``ic3net_b200.bptt.window_backward`` (pinned to the oracle in float64 by tests/test_bptt_manual.py) runs one step at a
time, last to first, from the recorded state entering each step, ``rec_h[t], rec_c[t]`` promoted to float64, with
``(dh, dc)`` chained from step t + 1.  The kernels read exactly these records, so the comparison isolates the backward
from any drift of the fp32 forward.  Observations come from the same snapshots the kernels read: the predator-prey
sparse pattern of ``s_loc[t]``, the traffic-junction block that ``ic3_tj_obs`` writes for ``s_tj*[t]``.

``oracle_grad_sum`` is the other yardstick: the float64 oracle replaying every env slot of a ``run_batch`` as one
reference process (teacher-forced with the GPU's actions) and summing the gradients over slots."""
import numpy as np
import torch

from ic3net_b200 import bptt

LOSS_KEYS = ("action_loss", "value_loss", "entropy")


def chain_one_step(P, G, spec, rec, state, adv, ret):
    """Backward of steps [0, T) as T one-step windows.  state(t) -> (h, c) entering step t; gradients are added to G.
    Returns the three loss sums."""
    T = rec["fresh"].shape[0]
    tot = dict.fromkeys(LOSS_KEYS, 0.0)
    dh = dc = None
    for t in reversed(range(T)):
        h0, c0 = state(t)
        dh, dc, st = bptt.window_backward(P, G, spec, rec, t, t + 1, h0, c0, adv, ret, dh, dc)
        for q in tot:
            tot[q] += st[q]
    return tot


def returns_and_advantages(tr):
    """(ret, adv) [T, B, N] float32, computed as Trainer.compute_grad_device does before it calls the kernels."""
    from ic3net_b200 import _lib
    b, args, e = tr._buf, tr.args, tr.env.env
    T, B, N = b["T"], e.nenvs, args.nagents
    ret = torch.empty(T, B, N, device=e.device)
    _lib.check(_lib.load().ic3_returns_scan(T, B, N, float(args.gamma), float(args.mean_ratio), b["reward"].data_ptr(),
                                            b["emask"].data_ptr(), b["mini"].data_ptr(), ret.data_ptr(),
                                            _lib.stream()))
    adv = ret - b["value"].view(T, B, N)
    if args.normalize_rewards:
        v = b["valid"].float().unsqueeze(-1)
        cnt = v.sum(0, keepdim=True) * N
        mean = (adv * v).sum((0, 2), keepdim=True) / cnt
        var = (((adv - mean) * v) ** 2).sum((0, 2), keepdim=True) / (cnt - 1)
        adv = (adv - mean) / var.sqrt()
    return ret, adv


def tj_record_obs(tr, t, k0, k1):
    """[k1 - k0, N, O] float32 traffic-junction observation of step t for env slots [k0, k1), written by ic3_tj_obs
    from the recorded state (Trainer._record_state)."""
    return tr._tj_record_obs(t, k0, k1)


def trainer_reference(tr, slots=None, heads_from_records=True):
    """Float64 gradient of every parameter (dict by name, device tensors) and the three loss sums of the batch the
    kernel trainer ``tr`` recorded.  ``slots = (k0, k1)`` restricts both to env slots [k0, k1) (slots are independent,
    so the full-batch result is the sum over any partition of the slots).  ``heads_from_records``: the heads' backward
    starts from the recorded log-probabilities and values, as the kernels' does; False re-evaluates the heads on the
    recorded h' in float64 instead, which adds the fp32 forward's rounding of those outputs to the difference."""
    assert tr.grad_kernels, "the reference reads the records of the BPTT kernel path"
    b, args, net, e = tr._buf, tr.args, tr.policy_net, tr.env.env
    B, N = e.nenvs, args.nagents
    k0, k1 = (0, B) if slots is None else slots
    s, rows = slice(k0, k1), slice(k0 * N, k1 * N)
    f64 = torch.float64
    ret, adv = returns_and_advantages(tr)
    P = {k: v.detach().to(f64) for k, v in net.named_parameters() if not k.startswith("hidd_encoder")}
    G = {k: torch.zeros_like(v) for k, v in P.items()}
    spec = bptt.Spec(N, args.hid_size, len(args.naction_heads), bool(args.hard_attn) and bool(args.commnet),
                     getattr(args, "comm_mode", "avg") == "avg", bool(args.comm_mask_zero), args.value_coeff, args.entr,
                     args.detach_gap, args.max_steps)
    if tr.is_tj:
        def obs(t):
            return tj_record_obs(tr, t, k0, k1).reshape((k1 - k0) * N, -1).to(f64)
    else:
        def obs(t):
            idx, val = tr._pp_sparse_obs(b["s_loc"][t, s])
            return idx, val.to(f64)
    rec = dict(fresh=b["s_fresh"][:, s], comm=b["s_comm"][:, s], alive=b["s_alive"][:, s], t_ep=b["s_tep"][:, s],
               action=b["action"][:, s], alive_post=b["ralive"][:, s], valid=b["valid"][:, s], obs=obs)
    if heads_from_records:
        rec.update(value=b["value"][:, rows], logp=b["logp"][:, s])

    def state(t):
        # slots starting an episode enter the step with a zero state whatever the record holds (rec_h[0] is never
        # written: every slot starts fresh), so they are zeroed here rather than multiplied by zero
        fresh = b["s_fresh"][t, s].bool().repeat_interleave(N).unsqueeze(1)
        h, c = b["rec_h"][t, rows].to(f64), b["rec_c"][t, rows].to(f64)
        return h.masked_fill(fresh, 0.0), c.masked_fill(fresh, 0.0)

    tot = chain_one_step(P, G, spec, rec, state, adv[:, s].to(f64), ret[:, s].to(f64))
    return G, tot


def heads_abs_sums(tr):
    """{heads.m.weight / bias: sum over rows and steps of |term|} of the action heads' gradients (float64), from the
    same records the kernels read.  The two-logit communication head's gradient cancels to a small fraction of these
    sums, so its fp32 per-row terms carry an error of a few units of 2^-24 of the SUM, not of the result."""
    b, args = tr._buf, tr.args
    T, B, N = b["T"], tr.env.env.nenvs, args.nagents
    R = B * N
    f64 = torch.float64
    _, adv = returns_and_advantages(tr)
    out = {}
    for t in range(T):
        a = (-adv[t].reshape(R, 1) * b["ralive"][t].reshape(R, 1)).to(f64)
        vrow = b["valid"][t].to(f64).repeat_interleave(N).unsqueeze(1)
        h2 = b["rec_h"][t + 1].to(f64).abs()
        lp_all = b["logp"][t].reshape(R, -1).to(f64)
        act = b["action"][t].long().reshape(R, -1)
        off = 0
        for m, na in enumerate(args.naction_heads):
            lp = lp_all[:, off:off + na]
            p = lp.exp()
            g = a * (torch.zeros_like(p).scatter_(1, act[:, m:m + 1], 1.0) - p)
            if args.entr > 0:
                g = g + args.entr * p * (lp - (p * lp).sum(1, keepdim=True)) * vrow
            g = g.abs()
            for key, v in (("heads.%d.bias" % m, g.sum(0)), ("heads.%d.weight" % m, g.t() @ h2)):
                out[key] = out[key] + v if key in out else v
            off += na
    return out


def oracle_grad_sum(args, z, p, act, valid, seed, id0, quota, T):
    """Float64 oracle gradient (dict by name, numpy; None for unused parameters) and loss sums of a run_batch whose
    slots played with Philox streams (seed, id0 + b), teacher-forced with the GPU's actions act [T, B, N, heads]: every
    slot is one reference process playing whole episodes until it holds >= quota steps.  Also returns the number
    of steps the slots played."""
    from helpers import make_oracle_env, tj_tables
    from oracle import grad as ograd
    from oracle.rollout import run_episode
    is_tj = args.env_name == "traffic_junction"
    want, wstat = None, dict.fromkeys(LOSS_KEYS, 0.0)
    nsteps = 0
    for b in range(act.shape[1]):
        orc = make_oracle_env(args, tj_tables(z) if is_tj else None)
        eps, t0, k = [], 0, 0
        while t0 < quota:                    # trainer.py:231: whole episodes until the slot holds >= batch_size steps
            ep = run_episode(orc, p, args, seed, id0 + b, epoch=0, tick0=t0, episode=k, forced_actions=act[t0:, b])
            eps.append(ep)
            t0 += ep["num_steps"]
            k += 1
        assert t0 <= T and valid[:t0, b].all() and not valid[t0:, b].any(), (b, t0)
        nsteps += t0
        g, st, _ = ograd.compute_grad(p, eps, args)
        want = g if want is None else {q: (want[q] + g[q] if g[q] is not None else None) for q in g}
        for q in wstat:
            wstat[q] += st[q]
    return want, wstat, nsteps


def max_rel_err(got, want):
    """max |got - want| / max |want| (inf when want is all zero and got is not, 0 when both are)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    d, m = np.abs(got - want).max(), np.abs(want).max()
    return d / m if m > 0 else (0.0 if d == 0 else np.inf)
