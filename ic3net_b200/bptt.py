"""Explicit backward pass (BPTT) of the rollout loss over the trainer's lock-step record buffers.

``Trainer.compute_grad`` (reference trainer.py:128-225) needs d(loss)/d(parameters) through the recurrent policy.
This module states that gradient for the one-pass LSTM CommNet / IC3Net with the hand-derived per-step formulas
(spelled out and pinned to the reference's gradients in ``oracle/bptt.py``): a window is re-run forward without a
graph, keeping only the activations the backward needs, then walked backwards with batched GEMMs -- exactly the
arithmetic the hand-written BPTT kernels (csrc/bptt_tc.cu) perform.  No ``Trainer`` backend runs it: it is the float64
reference the tests compare the kernels against, in plain torch ops on whatever device / dtype the records live on.

Step t of the lock-step batch (rows = B env slots x N agents; ``fresh`` marks slots that start an episode):

    h, c   <- 0 for fresh slots (trainer.py:50-51)              alive <- 1, comm_action <- 0 for fresh slots
    x      = encoder(obs)                                        (comm.py:119)
    g      = alive * comm_action        (hard attention)         tot = sum_j g_j h_j,  den = n_alive - 1 (avg mode)
    S_k    = g_k (tot - g_k h_k) / den                           (comm.py:181-205)
    u      = x + S W_c^T + b_c ;  a = u W_ih^T + b_ih + h W_hh^T + b_hh ;  LSTM cell -> (h', c')
    value  = h' w_v + b_v ;  logp^m = log_softmax(h' W_m^T + b_m)
    loss  += sum alive_post [ -A logp(action) + value_coeff (value - R)^2 ] + entr * sum logp exp(logp)
    (h', c') are detached for slots with (t_ep + 1) % detach_gap == 0  (trainer.py:56-60)
"""
import torch

PARAM_KEYS = ("encoder.weight", "encoder.bias", "C_modules.0.weight", "C_modules.0.bias", "f_module.weight_ih",
              "f_module.weight_hh", "f_module.bias_ih", "f_module.bias_hh", "value_head.weight", "value_head.bias")


class Spec(object):
    """Static facts of the policy / loss the backward needs."""

    def __init__(self, nagents, hid_size, nheads, hard_attn, comm_avg=True, comm_mask_zero=False, value_coeff=0.01,
                 entr=0.0, detach_gap=10000, max_steps=20):
        self.N, self.H, self.nheads = int(nagents), int(hid_size), int(nheads)
        self.hard, self.comm_avg, self.comm_mask_zero = bool(hard_attn), bool(comm_avg), bool(comm_mask_zero)
        self.value_coeff, self.entr = float(value_coeff), float(entr)
        self.detach = int(detach_gap) if int(detach_gap) <= int(max_steps) else 0      # 0: never detaches


def encode(P, obs):
    """x = encoder(obs); obs is a dense [R, O] tensor or a sparse (index [R, K], value [R, K]) pair."""
    if isinstance(obs, tuple):
        idx, val = obs
        return (P["encoder.weight"].t()[idx] * val.unsqueeze(-1)).sum(1) + P["encoder.bias"]
    return obs @ P["encoder.weight"].t() + P["encoder.bias"]


def _encoder_grad(G, obs, du):
    if isinstance(obs, tuple):                     # scatter-add of du rows, weighted by the feature values
        idx, val = obs
        contrib = (du.unsqueeze(1) * val.unsqueeze(-1)).reshape(-1, du.shape[1])       # [R*K, H]
        gT = torch.zeros(G["encoder.weight"].shape[1], du.shape[1], dtype=du.dtype, device=du.device)
        gT.index_add_(0, idx.reshape(-1), contrib)
        G["encoder.weight"] += gT.t()
    else:
        G["encoder.weight"] += du.t() @ obs
    G["encoder.bias"] += du.sum(0)


def _forward(P, spec, rec, t, h, c):
    """One step without a graph; returns (h', c', cache)."""
    N, H = spec.N, spec.H
    B = rec["fresh"].shape[1]
    dt = h.dtype
    fresh = rec["fresh"][t].bool()                                                    # [B]
    keep = (~fresh).to(dt).repeat_interleave(N).unsqueeze(1)                          # [R, 1]
    h, c = h * keep, c * keep
    obs = rec["obs"](t)
    x = encode(P, obs)
    f2 = fresh.unsqueeze(1)
    alive = torch.where(f2, torch.ones_like(rec["alive"][t]), rec["alive"][t]).to(dt)          # comm.py:99-112
    n_alive = alive.sum(1, keepdim=True)
    g = alive
    if spec.hard:
        g = g * torch.where(f2, torch.zeros_like(rec["comm"][t]), rec["comm"][t]).to(dt)       # comm.py:171-175
    if spec.comm_avg:
        den = torch.where(n_alive > 1, n_alive - 1, torch.ones_like(n_alive))
    else:
        den = torch.ones_like(n_alive)
    gs = (g / den).reshape(B * N, 1)                   # g_k / den
    gr = g.reshape(B * N, 1)
    if spec.comm_mask_zero:
        S = torch.zeros_like(h)
    else:
        tot = (gr * h).view(B, N, H).sum(1, keepdim=True).expand(B, N, H).reshape(B * N, H)
        S = gs * (tot - gr * h)
    u = x + S @ P["C_modules.0.weight"].t() + P["C_modules.0.bias"]
    a = (u @ P["f_module.weight_ih"].t() + P["f_module.bias_ih"] + h @ P["f_module.weight_hh"].t()
         + P["f_module.bias_hh"])
    si, sf, tg, so = torch.sigmoid(a[:, :H]), torch.sigmoid(a[:, H:2 * H]), torch.tanh(a[:, 2 * H:3 * H]), \
        torch.sigmoid(a[:, 3 * H:])
    c2 = sf * c + si * tg
    tc = torch.tanh(c2)
    h2 = so * tc
    cache = dict(keep=keep, obs=obs, h=h, c=c, gs=gs, gr=gr, S=S, u=u, si=si, sf=sf, tg=tg, so=so, tc=tc, h2=h2)
    return h2, c2, cache


def window_backward(P, G, spec, rec, t0, t1, h0, c0, adv, ret, dh_in=None, dc_in=None):
    """Gradient contribution of steps [t0, t1) accumulated into ``G`` (dict like ``P``, same shapes).

    P: parameters by state_dict name (``heads.m.weight/bias`` for m < nheads);  rec: dict with ``fresh [T,B]``,
    ``comm [T,B,N]``, ``alive [T,B,N]`` (inputs of each policy step), ``t_ep [T,B]``, ``action [T,B,N,nheads]``,
    ``alive_post [T,B,N]`` and ``obs`` = callable t -> dense [R,O] or (index, value); optionally ``valid [T,B]`` and
    the rollout's recorded ``value [T,R]`` / ``logp [T,B,N,sum of head sizes]``, from which the heads' backward then
    starts instead of re-evaluating the heads on h' (the BPTT kernels read them that way);  adv, ret: [T,B,N];
    (h0, c0): state entering step t0;  (dh_in, dc_in): d loss / d (h', c') of step t1-1 coming from later steps.
    Returns (d loss / d h0, d loss / d c0, stats dict of python floats)."""
    N, H = spec.N, spec.H
    B = rec["fresh"].shape[1]
    R = B * N
    with torch.no_grad():
        caches, h, c = [], h0, c0
        for t in range(t0, t1):
            h, c, ch = _forward(P, spec, rec, t, h, c)
            caches.append(ch)
        dt = h.dtype
        dh = torch.zeros(R, H, dtype=dt, device=h.device) if dh_in is None else dh_in
        dc = torch.zeros(R, H, dtype=dt, device=h.device) if dc_in is None else dc_in
        st = dict(action_loss=0.0, value_loss=0.0, entropy=0.0)
        a_l = torch.zeros((), dtype=dt, device=h.device)
        v_l = torch.zeros((), dtype=dt, device=h.device)
        ent = torch.zeros((), dtype=dt, device=h.device)
        W_ih, W_hh, W_c = P["f_module.weight_ih"], P["f_module.weight_hh"], P["C_modules.0.weight"]
        for t in reversed(range(t0, t1)):
            ch = caches[t - t0]
            h2 = ch["h2"]
            if spec.detach:                                                            # trainer.py:56-60
                cut = (((rec["t_ep"][t] + 1) % spec.detach) == 0).repeat_interleave(N).unsqueeze(1)
                dh = torch.where(cut, torch.zeros_like(dh), dh)
                dc = torch.where(cut, torch.zeros_like(dc), dc)
            alive_post = rec["alive_post"][t].to(dt).reshape(R)
            A, Rt = adv[t].reshape(R).to(dt), ret[t].reshape(R).to(dt)
            act = rec["action"][t].long().reshape(R, -1)
            # value head (from the rollout's recorded outputs when given, as the BPTT kernels read them)
            if "value" in rec:
                value = rec["value"][t].reshape(R).to(dt)
            else:
                value = (h2 @ P["value_head.weight"].t() + P["value_head.bias"])[:, 0]
            dv = 2.0 * spec.value_coeff * alive_post * (value - Rt)
            v_l += (((value - Rt) ** 2) * alive_post).sum()
            G["value_head.weight"] += (dv.unsqueeze(1) * h2).sum(0, keepdim=True)
            G["value_head.bias"] += dv.sum().reshape(1)
            dh = dh + dv.unsqueeze(1) * P["value_head.weight"]
            # action heads
            lp_taken = torch.zeros(R, dtype=dt, device=h.device)
            # slots that already completed their batch (trainer.py:231) contribute nothing, not even entropy
            vrow = rec["valid"][t].to(dt).repeat_interleave(N).unsqueeze(1) if "valid" in rec else 1.0
            off = 0
            for m in range(spec.nheads):
                Wm, bm = P["heads.%d.weight" % m], P["heads.%d.bias" % m]
                if "logp" in rec:
                    logp = rec["logp"][t].reshape(R, -1)[:, off:off + Wm.shape[0]].to(dt)
                else:
                    logp = torch.log_softmax(h2 @ Wm.t() + bm, dim=-1)
                off += Wm.shape[0]
                pm = logp.exp()
                am = act[:, m:m + 1]
                lp_taken += logp.gather(-1, am).squeeze(-1)
                onehot = torch.zeros_like(pm).scatter_(-1, am, 1.0)
                dlogit = (-A * alive_post).unsqueeze(1) * (onehot - pm)
                ent -= (logp * pm * vrow).sum()
                if spec.entr > 0:
                    Hm = -(pm * logp).sum(-1, keepdim=True)
                    dlogit = dlogit + spec.entr * pm * (logp + Hm) * vrow
                G["heads.%d.weight" % m] += dlogit.t() @ h2
                G["heads.%d.bias" % m] += dlogit.sum(0)
                dh = dh + dlogit @ Wm
            a_l += (-A * lp_taken * alive_post).sum()
            # LSTM cell
            si, sf, tg, so, tc = ch["si"], ch["sf"], ch["tg"], ch["so"], ch["tc"]
            do = dh * tc
            dc = dc + dh * so * (1.0 - tc * tc)
            da = torch.cat([dc * tg * si * (1.0 - si), dc * ch["c"] * sf * (1.0 - sf), dc * si * (1.0 - tg * tg),
                            do * so * (1.0 - so)], dim=1)
            dc_prev = dc * sf
            G["f_module.weight_ih"] += da.t() @ ch["u"]
            G["f_module.weight_hh"] += da.t() @ ch["h"]
            dab = da.sum(0)
            G["f_module.bias_ih"] += dab
            G["f_module.bias_hh"] += dab
            du = da @ W_ih
            dh_prev = da @ W_hh
            # communication: S_k = (g_k/den) (tot - g_k h_k)
            G["C_modules.0.weight"] += du.t() @ ch["S"]
            G["C_modules.0.bias"] += du.sum(0)
            if not spec.comm_mask_zero:
                dSs = (du @ W_c) * ch["gs"]
                dtot = dSs.view(B, N, H).sum(1, keepdim=True).expand(B, N, H).reshape(R, H)
                dh_prev = dh_prev + ch["gr"] * (dtot - ch["gr"] * dSs)
            _encoder_grad(G, ch["obs"], du)
            # through the episode-start reset of (h, c)
            dh, dc = dh_prev * ch["keep"], dc_prev * ch["keep"]
        st["action_loss"], st["value_loss"], st["entropy"] = float(a_l), float(v_l), float(ent)
    return dh, dc, st
