"""Float64 yardsticks for the non-recurrent tanh policies: models.MLP (models.py:8-36) and CommNet / IC3Net without
--recurrent (comm.py:114-131, 179-224) (TEST INFRASTRUCTURE).

``ff_oracle(model, passes, share)`` is a context in which the float64 oracle (oracle/policy.py, oracle/rollout.py,
oracle/grad.py, and the weights of oracle/gen_golden.py) runs these policies instead of the recurrent CommNet:
    x = tanh(encoder(obs)),  h_0 = x,  per pass i: S = gated mean of h_i,  h_{i+1} = tanh(x + f_i(h_i) + C_i(S))
    models.MLP: one pass with no communication, h = tanh(affine2(x) + x)
The value oracle steps through ``oracle.policy.forward_variant`` (x_tanh, h_from_x); the gradient oracle restates the
step with torch float64 autograd.  With share_weights the one f and C module's gradients are the sums over the passes,
as the reference's shared parameters get them.  Everything that calls the oracle inside the context --
``oracle.gen_golden.gen_grad_case`` writing the ``gradff_*`` fixtures from the unmodified reference
(scripts/gen_golden_ff.py), ``bptt_ref.oracle_grad_sum`` replaying a GPU batch -- then runs the non-recurrent policy.

``records_reference(tr)`` is the float64 backward of the batch a ``grad_impl='kernels_ff'`` trainer recorded: every step
re-run in float64 from the recorded env state and masks, differentiated by torch autograd, with the heads' backward
started from the recorded log-probs and values as the kernels' is."""
import contextlib

import numpy as np
import torch
import torch.nn.functional as F

from oracle import gen_golden, policy
from oracle import grad as ograd

_make_weights_1 = gen_golden.make_weights             # captured before any patching
LOSS_KEYS = ("action_loss", "value_loss", "entropy")


def make_weights(seed, obs_dim, hid, heads, comm_init="uniform", model="commnet", passes=1, share=False):
    """state_dict of models.MLP (affine1 / affine2 from the encoder's and the first comm module's draws) or of the
    non-recurrent CommNetMLP (encoder, f_modules.i from the hidd_encoder draw of seed + 1000 i, C_modules.i from the
    comm module's draw of seed + 1000 i; share_weights: every pass and f_module / C_module hold pass 0's weights)."""
    sd = _make_weights_1(seed, obs_dim, hid, heads, comm_init)
    out = {k: v for k, v in sd.items() if k.startswith("heads.") or k.startswith("value_head.")}
    if model == "mlp":
        out.update({"affine1.weight": sd["encoder.weight"], "affine1.bias": sd["encoder.bias"],
                    "affine2.weight": sd["C_modules.0.weight"], "affine2.bias": sd["C_modules.0.bias"]})
        return out
    out["encoder.weight"], out["encoder.bias"] = sd["encoder.weight"], sd["encoder.bias"]
    for i in range(passes):
        src = sd if (i == 0 or share) else _make_weights_1(seed + 1000 * i, obs_dim, hid, heads, comm_init)
        for k in ("weight", "bias"):
            out["f_modules.%d.%s" % (i, k)] = src["hidd_encoder." + k].copy()
            out["C_modules.%d.%s" % (i, k)] = src["C_modules.0." + k].copy()
    if share:
        for k in ("weight", "bias"):
            out["f_module." + k] = out["f_modules.0." + k].copy()
            out["C_module." + k] = out["C_modules.0." + k].copy()
    return out


def _names(p, model, passes):
    if model == "mlp":
        return "affine1", ["affine2"], None
    return "encoder", ["f_modules.%d" % i for i in range(passes)], ["C_modules.%d" % i for i in range(passes)]


def _forward_np(model, passes):
    def forward(params, obs, h, c, comm_action=None, alive=None, hard_attn=True, comm_mode="avg", comm_mask_zero=False):
        roles = policy.roles_of(params, "commnet" if model == "commnet" else "mlp", False, passes)
        lo, v, h2, _ = policy.forward_variant(roles, obs, h, None, comm_action, alive, hard_attn, comm_mode,
                                              comm_mask_zero or model == "mlp", passes, x_tanh=True, h_from_x=True)
        x = np.tanh(np.asarray(obs, dtype=np.float64) @ roles["enc"][0].T + roles["enc"][1])
        return lo, v, h2, c, x
    return forward


def step_torch(p, model, passes, x_pre, g, den, B, N, comm_mask_zero):
    """Differentiable non-recurrent step for B envs of N agents: x_pre [B*N, H] (encoder output before the tanh),
    g [B, N] comm gates, den [B, 1] mean denominators.  Returns h_P."""
    enc, fn, cn = _names(p, model, passes)
    x = torch.tanh(x_pre)
    hid = x
    H = x.shape[1]
    gg = g.unsqueeze(-1)
    for i in range(passes):
        h = hid @ p[fn[i] + ".weight"].t() + p[fn[i] + ".bias"]
        if cn is not None:
            if comm_mask_zero or N < 2:
                S = torch.zeros_like(hid)
            else:
                hv = hid.view(B, N, H)
                S = (gg * ((gg * hv).sum(1, keepdim=True) - gg * hv) / den.unsqueeze(-1)).reshape(B * N, H)
            h = h + S @ p[cn[i] + ".weight"].t() + p[cn[i] + ".bias"]
        hid = torch.tanh(x + h)
    return hid


def _forward_torch(model, passes):
    def forward(p, obs, h, c, comm_action, alive, hard_attn, comm_mode="avg", comm_mask_zero=False):
        n = obs.shape[0]
        enc = "affine1" if model == "mlp" else "encoder"
        alive_v = torch.ones(n, dtype=torch.float64) if alive is None else torch.as_tensor(alive, dtype=torch.float64)
        n_alive = float(alive_v.sum())
        g = alive_v.clone()
        if hard_attn:
            g = g * torch.as_tensor(comm_action, dtype=torch.float64)
        den = n_alive - 1 if (comm_mode == "avg" and n_alive > 1) else 1.0
        h2 = step_torch(p, model, passes, obs @ p[enc + ".weight"].t() + p[enc + ".bias"], g.view(1, n),
                        torch.full((1, 1), den, dtype=torch.float64), 1, n, comm_mask_zero)
        value = (h2 @ p["value_head.weight"].t() + p["value_head.bias"])[:, 0]
        logps, k = [], 0
        while "heads.%d.weight" % k in p:
            logps.append(torch.log_softmax(h2 @ p["heads.%d.weight" % k].t() + p["heads.%d.bias" % k], dim=-1))
            k += 1
        return logps, value, h2, c
    return forward


@contextlib.contextmanager
def ff_oracle(model="commnet", passes=1, share=False):
    saved = (policy.forward, ograd.forward_torch, ograd.compute_grad, gen_golden.make_weights)
    compute_grad_1 = ograd.compute_grad

    def compute_grad(params_np, episodes, args):
        g, st, extra = compute_grad_1(params_np, episodes, args)
        if share:                                  # one module per role: the sum of what every pass contributes
            for mod, alias in (("f_modules", "f_module"), ("C_modules", "C_module")):
                for k in ("weight", "bias"):
                    tot = sum(g["%s.%d.%s" % (mod, i, k)] for i in range(passes))
                    for key in ["%s.%d.%s" % (mod, i, k) for i in range(passes)] + ["%s.%s" % (alias, k)]:
                        g[key] = tot.copy()
        return g, st, extra

    policy.forward = _forward_np(model, passes)
    ograd.forward_torch = _forward_torch(model, passes)
    ograd.compute_grad = compute_grad
    gen_golden.make_weights = lambda seed, obs_dim, hid, heads, comm_init="uniform": make_weights(
        seed, obs_dim, hid, heads, comm_init, model, passes, share)
    try:
        yield
    finally:
        policy.forward, ograd.forward_torch, ograd.compute_grad, gen_golden.make_weights = saved


def records_reference(tr):
    """Float64 gradient of every parameter (dict by name, device tensors), the three loss sums, and the action heads'
    sums of |term| (the scale of their fp32 rounding) of the batch a kernels_ff trainer recorded."""
    from bptt_ref import returns_and_advantages, tj_record_obs
    b, args, net, e = tr._buf, tr.args, tr.policy_net, tr.env.env
    T, B, N = b["T"], e.nenvs, args.nagents
    R = B * N
    f64 = torch.float64
    model = "mlp" if hasattr(net, "affine1") else "commnet"
    passes = 1 if model == "mlp" else int(args.comm_passes)
    enc = "affine1" if model == "mlp" else "encoder"
    ret, adv = returns_and_advantages(tr)
    ret, adv = ret.to(f64).reshape(T, R), adv.to(f64).reshape(T, R)
    names = {id(q): n for n, q in net.named_parameters()}
    P = {n: q.detach().to(f64).requires_grad_(True) for n, q in net.named_parameters()}
    # the step addresses every pass's module by its list name: shared modules map to the one parameter
    p = dict(P)
    if model == "commnet":
        for i in range(passes):
            for k in ("weight", "bias"):
                p["f_modules.%d.%s" % (i, k)] = P[names[id(getattr(net.f_modules[i], k))]]
                p["C_modules.%d.%s" % (i, k)] = P[names[id(getattr(net.C_modules[i], k))]]
    G = {n: torch.zeros_like(q) for n, q in P.items()}
    hsum = {}
    hard = bool(args.hard_attn) and bool(args.commnet)
    comm_avg = getattr(args, "comm_mode", "avg") == "avg"
    cmz = bool(args.comm_mask_zero) or model == "mlp"
    nh = len(args.naction_heads)
    tot = dict.fromkeys(LOSS_KEYS, 0.0)
    plist = list(P.values())
    for t in range(T):
        if tr.is_tj:
            obs = tj_record_obs(tr, t, 0, B).reshape(R, -1).to(f64)
            x_pre = obs @ P[enc + ".weight"].t() + P[enc + ".bias"]
        else:
            idx, val = tr._pp_sparse_obs(b["s_loc"][t])
            x_pre = F.embedding_bag(idx, P[enc + ".weight"].t(), per_sample_weights=val.to(f64), mode="sum") + \
                P[enc + ".bias"]
        fresh = b["s_fresh"][t].bool().unsqueeze(1)
        alive = torch.where(fresh, torch.ones_like(b["s_alive"][t]), b["s_alive"][t]).to(f64)    # comm.py:99-112
        n_alive = alive.sum(1, keepdim=True)
        g = alive
        if hard:
            g = g * torch.where(fresh, torch.zeros_like(b["s_comm"][t]), b["s_comm"][t]).to(f64)  # comm.py:171-175
        den = torch.where(n_alive > 1, n_alive - 1, torch.ones_like(n_alive)) if comm_avg else torch.ones_like(n_alive)
        h = step_torch(p, model, passes, x_pre, g, den, B, N, cmz)
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
            ha = h.detach().abs()
            for key, term in (("heads.%d.weight" % m, dlogit.abs().t() @ ha), ("heads.%d.bias" % m, dlogit.abs().sum(0))):
                hsum[key] = hsum.get(key, 0.0) + term
        tot["action_loss"] += float((-adv[t] * lp_taken * alive_post).sum())
        out = torch.autograd.grad(sur, plist, allow_unused=True)
        for n_, gp in zip(P, out):
            if gp is not None:
                G[n_] += gp
    return G, tot, hsum
