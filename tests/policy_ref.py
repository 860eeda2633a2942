"""Float64 reference of one policy step for a whole batch of environments, and of its sampling.

``step_f64`` restates the recurrent (LSTM-cell) CommNet / IC3Net step of ``oracle.policy.forward_variant`` with batched
torch float64 ops over ``[B*N, .]`` rows, so that a full-size batch (81 920 rows) can be checked row by row on the device
that ran the kernels.  Episode starts follow ``ic3net_b200.bptt._forward`` (trainer.py:45-51): a ``fresh`` env enters the
step with a zero state, nobody in it talks and every agent counts as alive.

``philox_u24`` draws the 24-bit uniforms of ``oracle.philox.draw_u24`` for whole arrays of counters at once, and
``inverse_cdf`` is ``oracle.policy.sample_from_logp`` over whole arrays of rows.  tests/test_policy_ref.py pins all three to
the oracle."""
import numpy as np
import torch

from ic3net_b200 import bptt
from oracle import philox
from oracle import policy as opolicy


def params_f64(sd, passes=1, model="commnet", device="cpu"):
    """The parameter roles of ``oracle.policy.roles_of`` (recurrent branch) as float64 tensors on ``device``.  sd: a
    state_dict of numpy arrays or torch tensors with the reference's key names."""
    p = {k: (v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in sd.items()}
    r = opolicy.roles_of(opolicy.params_to_f64(p), model, True, passes)
    assert "lstm" in r, "step_f64 covers the LSTM cell"
    t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64), device=device)
    return dict(enc=tuple(t(a) for a in r["enc"]), C=[(t(w), t(b)) for w, b in r["C"]],
                lstm=tuple(t(a) for a in r["lstm"]), value=tuple(t(a) for a in r["value"]),
                heads=[(t(w), t(b)) for w, b in r["heads"]])


def step_f64(params, obs, h, c, comm, alive, fresh, *, nagents, passes=1, hard_attn=True, comm_mode="avg",
             comm_mask_zero=False):
    """One policy step of B envs x N agents in float64 (comm.py:134-244 with ``passes`` comm rounds).

    params: ``params_f64``;  obs: the observation as a dense [R, O] tensor or a sparse (index [R, K], value [R, K]) pair
    (``bptt.encode``);  h, c: [R, H] entering the step;
    comm, alive: [B, N] 0/1 (None: comm 0 / everybody alive);  fresh: [B] 0/1 or None.
    Returns (h' [R, H], c' [R, H], value [R], [log-probs [R, na] per head])."""
    N = int(nagents)
    R, H = h.shape
    B = R // N
    assert B * N == R
    dev, f64 = h.device, torch.float64
    fr = torch.zeros(B, dtype=torch.bool, device=dev) if fresh is None else torch.as_tensor(fresh, device=dev).bool()
    rows = fr.repeat_interleave(N).unsqueeze(1)
    # masked_fill, not a product: the state a fresh slot "enters" with may be anything, NaN included
    h = h.to(f64).masked_fill(rows, 0.0)
    c = c.to(f64).masked_fill(rows, 0.0)
    x = bptt.encode({"encoder.weight": params["enc"][0], "encoder.bias": params["enc"][1]}, obs)
    f2 = fr.unsqueeze(1)
    al = torch.ones(B, N, dtype=f64, device=dev) if alive is None else torch.as_tensor(alive, device=dev).to(f64)
    al = torch.where(f2, torch.ones_like(al), al)                                     # comm.py:99-112
    n_alive = al.sum(1, keepdim=True)
    g = al
    if hard_attn:
        cm = torch.zeros(B, N, dtype=f64, device=dev) if comm is None else torch.as_tensor(comm, device=dev).to(f64)
        g = g * torch.where(f2, torch.zeros_like(cm), cm)                            # comm.py:171-175
    if comm_mode == "avg":
        den = torch.where(n_alive > 1, n_alive - 1, torch.ones_like(n_alive))          # comm.py:194-196
    else:
        den = torch.ones_like(n_alive)
    gg = g.unsqueeze(-1)
    w_ih, w_hh, b_ih, b_hh = params["lstm"]
    hid = h
    for ps in range(passes):
        if comm_mask_zero:
            S = torch.zeros_like(hid)
        else:                                                                        # comm.py:181-205
            hv = hid.view(B, N, H)
            tot = (gg * hv).sum(1, keepdim=True)
            S = (gg * (tot - gg * hv) / den.unsqueeze(-1)).reshape(R, H)
        cw, cb = params["C"][ps]
        a = (x + S @ cw.t() + cb) @ w_ih.t() + b_ih + hid @ w_hh.t() + b_hh              # comm.py:206-218
        gi, gf, gq, go = (a[:, k * H:(k + 1) * H] for k in range(4))
        c = torch.sigmoid(gf) * c + torch.sigmoid(gi) * torch.tanh(gq)
        hid = torch.sigmoid(go) * torch.tanh(c)
    vw, vb = params["value"]
    value = (hid @ vw.t() + vb)[:, 0]
    logps = [torch.log_softmax(hid @ w.t() + b, dim=-1) for w, b in params["heads"]]
    return hid, c, value, logps


def philox_u24(seed, env_ids, ticks, stream, index):
    """Four 24-bit draws per counter (env_id, tick, stream, index), broadcast over numpy arrays: [..., 4] int64."""
    e, t, s, i = np.broadcast_arrays(*(np.asarray(v, dtype=np.uint64) for v in (env_ids, ticks, stream, index)))
    ctr = np.stack([e, t, s, i], axis=-1)
    return (philox.philox4x32(ctr, philox.split_seed(seed)) >> np.uint32(8)).astype(np.int64)


def inverse_cdf(logp, u24):
    """Inverse-CDF sampling of every row: logp [M, na] (numpy / torch), u24 [M] integers.  Returns numpy
    (action [M], margin [M]): the smallest a with sum_{i<=a} exp(logp_i) > u24 * 2^-24, else na - 1, and the distance of
    the uniform to the nearest inner CDF edge (1 for a single action), as ``oracle.policy.sample_from_logp``."""
    lp = logp.detach().cpu().numpy() if torch.is_tensor(logp) else np.asarray(logp)
    cdf = np.cumsum(np.exp(lp.astype(np.float64)), axis=-1)
    u = np.asarray(u24, dtype=np.float64).reshape(-1, 1) * 2.0 ** -24
    na = cdf.shape[-1]
    above = cdf > u
    act = np.where(above.any(-1), above.argmax(-1), na - 1)
    margin = np.abs(cdf[:, :-1] - u).min(-1) if na > 1 else np.ones(cdf.shape[0])
    return act.astype(np.int64), margin
