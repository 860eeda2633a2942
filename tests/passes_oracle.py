"""Float64 yardsticks for CommNet / IC3Net with comm_passes > 1 and share_weights (TEST INFRASTRUCTURE).

``passes_oracle(passes, share)`` is a context in which the float64 oracle (oracle/policy.py, oracle/rollout.py,
oracle/grad.py, and the weights of oracle/gen_golden.py) follows comm.py:179-218 with ``passes`` comm rounds: the value
oracle steps through ``oracle.policy.forward_variant``, the gradient oracle restates the same rounds with torch
float64 autograd, and with share_weights the gradients of the one C module (``C_module`` and every ``C_modules.i``) are
the sum over the passes, as the reference's shared parameter gets them.  Everything that calls the oracle inside the
context -- ``oracle.gen_golden.gen_grad_case`` writing the ``gradpasses_*`` fixtures from the unmodified reference
(scripts/gen_golden_passes.py), ``bptt_ref.oracle_grad_sum`` replaying a GPU batch -- then runs the multi-pass policy.

``records_reference(tr)`` is the float64 backward of the batch a kernel trainer recorded, extended to passes: one step at
a time, last to first, from the recorded state entering the step, with every comm pass re-run in float64 and
differentiated by torch autograd; the heads' backward starts from the recorded values / log-probs, as the kernels'
does."""
import contextlib

import numpy as np
import torch

from oracle import gen_golden, policy
from oracle import grad as ograd

_make_weights_1 = gen_golden.make_weights          # the one-pass weights, captured before any patching
LOSS_KEYS = ("action_loss", "value_loss", "entropy")


def make_weights(seed, obs_dim, hid, heads, comm_init="uniform", passes=1, share=False):
    """oracle.gen_golden.make_weights plus C_modules.1 .. P-1 (from seeds seed + 1000 i); with share_weights every
    C_modules.i and C_module hold the weights of C_modules.0 (state_dict keys of comm.py:76-81)."""
    sd = _make_weights_1(seed, obs_dim, hid, heads, comm_init)
    for i in range(1, passes):
        src = sd if share else _make_weights_1(seed + 1000 * i, obs_dim, hid, heads, comm_init)
        for k in ("weight", "bias"):
            sd["C_modules.%d.%s" % (i, k)] = src["C_modules.0.%s" % k].copy()
    if share:
        for k in ("weight", "bias"):
            sd["C_module." + k] = sd["C_modules.0." + k].copy()
    return sd


def _c_keys(passes, share, k):
    return ["C_modules.%d.%s" % (i, k) for i in range(passes)] + (["C_module." + k] if share else [])


def _forward_np(passes):
    def forward(params, obs, h, c, comm_action=None, alive=None, hard_attn=True, comm_mode="avg", comm_mask_zero=False):
        roles = policy.roles_of(params, "commnet", True, passes)
        lo, v, h2, c2 = policy.forward_variant(roles, obs, h, c, comm_action, alive, hard_attn, comm_mode,
                                               comm_mask_zero, passes)
        x = np.asarray(obs, dtype=np.float64) @ params["encoder.weight"].T + params["encoder.bias"]
        return lo, v, h2, c2, x
    return forward


def _forward_torch(passes):
    def forward(p, obs, h, c, comm_action, alive, hard_attn, comm_mode="avg", comm_mask_zero=False):
        n, H = h.shape
        x = obs @ p["encoder.weight"].t() + p["encoder.bias"]
        alive_v = torch.ones(n, dtype=torch.float64) if alive is None else torch.as_tensor(alive, dtype=torch.float64)
        n_alive = float(alive_v.sum())
        g = alive_v.clone()
        if hard_attn:
            g = g * torch.as_tensor(comm_action, dtype=torch.float64)
        scale = 1.0 / (n_alive - 1) if (comm_mode == "avg" and n_alive > 1) else 1.0
        mask = (1.0 - torch.eye(n, dtype=torch.float64)) * g[:, None] * g[None, :] * scale    # [src, dst]
        for i in range(passes):                                                               # comm.py:179
            S = torch.zeros_like(h) if comm_mask_zero else mask.t() @ h
            cvec = S @ p["C_modules.%d.weight" % i].t() + p["C_modules.%d.bias" % i]
            gates = ((x + cvec) @ p["f_module.weight_ih"].t() + p["f_module.bias_ih"]
                     + h @ p["f_module.weight_hh"].t() + p["f_module.bias_hh"])
            gi, gf, gg, go = (gates[:, k * H:(k + 1) * H] for k in range(4))
            c = torch.sigmoid(gf) * c + torch.sigmoid(gi) * torch.tanh(gg)
            h = torch.sigmoid(go) * torch.tanh(c)
        value = (h @ p["value_head.weight"].t() + p["value_head.bias"])[:, 0]
        logps, k = [], 0
        while "heads.%d.weight" % k in p:
            logps.append(torch.log_softmax(h @ p["heads.%d.weight" % k].t() + p["heads.%d.bias" % k], dim=-1))
            k += 1
        return logps, value, h, c
    return forward


@contextlib.contextmanager
def passes_oracle(passes, share=False):
    saved = (policy.forward, ograd.forward_torch, ograd.compute_grad, gen_golden.make_weights)
    compute_grad_1 = ograd.compute_grad

    def compute_grad(params_np, episodes, args):
        g, st, extra = compute_grad_1(params_np, episodes, args)
        if share:                                  # one parameter: the sum of what every pass contributes
            for k in ("weight", "bias"):
                tot = sum(g["C_modules.%d.%s" % (i, k)] for i in range(passes))
                for key in _c_keys(passes, share, k):
                    g[key] = tot.copy()
        return g, st, extra

    policy.forward = _forward_np(passes)
    ograd.forward_torch = _forward_torch(passes)
    ograd.compute_grad = compute_grad
    gen_golden.make_weights = lambda seed, obs_dim, hid, heads, comm_init="uniform": make_weights(
        seed, obs_dim, hid, heads, comm_init, passes, share)
    try:
        yield
    finally:
        policy.forward, ograd.forward_torch, ograd.compute_grad, gen_golden.make_weights = saved


def records_reference(tr):
    """Float64 gradient of every parameter (dict by name, device tensors) and the three loss sums of the batch the kernel
    trainer ``tr`` recorded, comm_passes >= 1 (share_weights: one C module, named as in named_parameters)."""
    from bptt_ref import returns_and_advantages, tj_record_obs
    from ic3net_b200 import bptt
    assert tr.grad_kernels and "rec_h" in tr._buf
    b, args, net, e = tr._buf, tr.args, tr.policy_net, tr.env.env
    T, B, N, H = b["T"], e.nenvs, args.nagents, args.hid_size
    R = B * N
    f64 = torch.float64
    passes = int(args.comm_passes)
    ret, adv = returns_and_advantages(tr)
    ret, adv = ret.to(f64).reshape(T, R), adv.to(f64).reshape(T, R)
    names = {id(p): n for n, p in net.named_parameters()}
    P = {n: p.detach().to(f64).requires_grad_(True) for n, p in net.named_parameters() if not n.startswith("hidd_")}
    G = {n: torch.zeros_like(p) for n, p in P.items()}
    Cw = [P[names[id(m.weight)]] for m in net.C_modules]
    Cb = [P[names[id(m.bias)]] for m in net.C_modules]
    W_ih, W_hh = P["f_module.weight_ih"], P["f_module.weight_hh"]
    b_ih, b_hh = P["f_module.bias_ih"], P["f_module.bias_hh"]
    nh = len(args.naction_heads)
    hard = bool(args.hard_attn) and bool(args.commnet)
    comm_avg = getattr(args, "comm_mode", "avg") == "avg"
    detach = int(args.detach_gap) if int(args.detach_gap) <= int(args.max_steps) else 0
    dh = torch.zeros(R, H, dtype=f64, device=e.device)
    dc = torch.zeros_like(dh)
    tot = dict.fromkeys(LOSS_KEYS, 0.0)
    plist = list(P.values())
    for t in reversed(range(T)):
        fresh = b["s_fresh"][t].bool()
        frow = fresh.repeat_interleave(N).unsqueeze(1)
        h0 = b["rec_h"][t].to(f64).requires_grad_(True)
        c0 = b["rec_c"][t].to(f64).requires_grad_(True)
        h = torch.where(frow, torch.zeros_like(h0), h0)                   # trainer.py:50-51
        c = torch.where(frow, torch.zeros_like(c0), c0)
        if tr.is_tj:
            obs = tj_record_obs(tr, t, 0, B).reshape(R, -1).to(f64)
        else:
            idx, val = tr._pp_sparse_obs(b["s_loc"][t])
            obs = (idx, val.to(f64))
        x = bptt.encode(P, obs)
        f2 = fresh.unsqueeze(1)
        alive = torch.where(f2, torch.ones_like(b["s_alive"][t]), b["s_alive"][t]).to(f64)     # comm.py:99-112
        n_alive = alive.sum(1, keepdim=True)
        g = alive
        if hard:
            g = g * torch.where(f2, torch.zeros_like(b["s_comm"][t]), b["s_comm"][t]).to(f64)  # comm.py:171-175
        den = torch.where(n_alive > 1, n_alive - 1, torch.ones_like(n_alive)) if comm_avg else torch.ones_like(n_alive)
        gs, gr = (g / den).reshape(R, 1), g.reshape(R, 1)
        for i in range(passes):                                            # comm.py:179-218
            if args.comm_mask_zero:
                S = torch.zeros_like(h)
            else:
                tsum = (gr * h).view(B, N, H).sum(1, keepdim=True).expand(B, N, H).reshape(R, H)
                S = gs * (tsum - gr * h)
            a = (x + S @ Cw[i].t() + Cb[i]) @ W_ih.t() + b_ih + h @ W_hh.t() + b_hh
            gi, gf, gq, go = (a[:, k * H:(k + 1) * H] for k in range(4))
            c = torch.sigmoid(gf) * c + torch.sigmoid(gi) * torch.tanh(gq)
            h = torch.sigmoid(go) * torch.tanh(c)
        # d loss / d (value, logits) from the recorded outputs (trainer.py:186-220), as constants
        alive_post = b["ralive"][t].to(f64).reshape(R)
        vrow = b["valid"][t].to(f64).repeat_interleave(N).unsqueeze(1)
        value = b["value"][t].to(f64).reshape(R)
        dv = 2.0 * args.value_coeff * alive_post * (value - ret[t])
        tot["value_loss"] += float((((value - ret[t]) ** 2) * alive_post).sum())
        sur = (dv * (h @ P["value_head.weight"].t() + P["value_head.bias"])[:, 0]).sum()
        lp_all = b["logp"][t].reshape(R, -1).to(f64)
        act = b["action"][t].long().reshape(R, -1)
        lp_taken = torch.zeros(R, dtype=f64, device=e.device)
        off = 0
        for m in range(nh):
            na = args.naction_heads[m]
            lp = lp_all[:, off:off + na]
            off += na
            pm = lp.exp()
            lp_taken += lp.gather(-1, act[:, m:m + 1]).squeeze(-1)
            dlogit = (-adv[t] * alive_post).unsqueeze(1) * (torch.zeros_like(pm).scatter_(-1, act[:, m:m + 1], 1.0) - pm)
            tot["entropy"] -= float((lp * pm * vrow).sum())
            if args.entr > 0:
                Hm = -(pm * lp).sum(-1, keepdim=True)
                dlogit = dlogit + args.entr * pm * (lp + Hm) * vrow
            sur = sur + (dlogit * (h @ P["heads.%d.weight" % m].t() + P["heads.%d.bias" % m])).sum()
        tot["action_loss"] += float((-adv[t] * lp_taken * alive_post).sum())
        if detach:                                                         # trainer.py:56-60: (h', c') detached
            cut = (((b["s_tep"][t] + 1) % detach) == 0).repeat_interleave(N).unsqueeze(1)
            dh = torch.where(cut, torch.zeros_like(dh), dh)
            dc = torch.where(cut, torch.zeros_like(dc), dc)
        L = sur + (h * dh).sum() + (c * dc).sum()
        out = torch.autograd.grad(L, [h0, c0] + plist, allow_unused=True)
        dh, dc = out[0].detach(), out[1].detach()
        for n_, gp in zip(P, out[2:]):
            if gp is not None:
                G[n_] += gp
    return G, tot
