"""CPU tests (float64) of ic3net_b200/bptt.py -- the explicit backward pass over lock-step record buffers -- against
the autograd oracle (oracle/grad.py, itself pinned to the reference's Trainer.compute_grad): several env slots with
episode boundaries at different steps, windows chained through (dh, dc), detach gaps, alive masks, entropy term."""
import numpy as np
import pytest
import torch

from helpers import golden_names, load_golden, make_oracle_env, ns, tj_tables
from oracle import grad as ograd
from oracle import policy as opolicy
from oracle.gen_golden import make_weights
from oracle.rollout import run_episode

from ic3net_b200 import bptt


def _lockstep_records(name, B, T, seed=4242, id0=11):
    meta, z = load_golden(name)
    args = ns(meta["args"])
    is_tj = args.env_name == "traffic_junction"
    sd = make_weights(meta["weights_seed"], meta["obs_dim"], args.hid_size, meta["heads"], args.comm_init)
    p = opolicy.params_to_f64(sd)
    N, nh = args.nagents, len(meta["heads"])
    O = meta["obs_dim"]
    rec = dict(fresh=np.zeros((T, B), np.uint8), comm=np.zeros((T, B, N), np.int64), alive=np.ones((T, B, N)),
               t_ep=np.zeros((T, B), np.int64), action=np.zeros((T, B, N, nh), np.int64),
               alive_post=np.zeros((T, B, N)), obs=np.zeros((T, B, N, O)))
    adv, ret = np.zeros((T, B, N)), np.zeros((T, B, N))
    want, wstat = None, dict(action_loss=0.0, value_loss=0.0, entropy=0.0)
    for b in range(B):
        env = make_oracle_env(args, tj_tables(z) if is_tj else None)
        eps, t0, k = [], 0, 0
        while t0 < T:
            ep = run_episode(env, p, args, seed, id0 + b, epoch=0, tick0=t0, episode=k,
                             max_steps=min(args.max_steps, T - t0))
            for tt in range(ep["num_steps"]):
                t = t0 + tt
                rec["fresh"][t, b] = tt == 0
                rec["comm"][t, b] = ep["comm_in"][tt]
                rec["alive"][t, b] = ep["alive_in"][tt]
                rec["t_ep"][t, b] = tt
                rec["action"][t, b] = ep["act"][tt]
                rec["alive_post"][t, b] = ep["alive"][tt]
                rec["obs"][t, b] = ep["obs"][tt]
            eps.append(ep)
            t0 += ep["num_steps"]
            k += 1
        g, st, extra = ograd.compute_grad(p, eps, args)           # one slot = one reference process
        adv[:, b], ret[:, b] = extra["adv"], extra["returns"]
        want = g if want is None else {q: (want[q] + g[q] if g[q] is not None else None) for q in g}
        for q in wstat:
            wstat[q] += st[q]
    return meta, args, p, rec, adv, ret, want, wstat


def _run_manual(args, meta, p, rec, adv, ret, W, sparse=False):
    N, H, nh = args.nagents, args.hid_size, len(meta["heads"])
    T, B = rec["fresh"].shape
    P = {k: torch.tensor(v, dtype=torch.float64) for k, v in p.items()}
    G = {k: torch.zeros_like(v) for k, v in P.items()}
    spec = bptt.Spec(N, H, nh, bool(args.hard_attn) and bool(args.commnet), getattr(args, "comm_mode", "avg") == "avg",
                     bool(args.comm_mask_zero), args.value_coeff, args.entr, args.detach_gap, args.max_steps)
    tobs = torch.tensor(rec["obs"]).reshape(T, B * N, -1)

    def obs_fn(t):
        o = tobs[t]
        if not sparse:
            return o
        K = int((o != 0).sum(1).max())
        idx = torch.zeros(o.shape[0], K, dtype=torch.long)
        val = torch.zeros(o.shape[0], K, dtype=torch.float64)
        for r in range(o.shape[0]):
            nz = torch.nonzero(o[r]).flatten()
            idx[r, :len(nz)] = nz
            val[r, :len(nz)] = o[r, nz]
        return idx, val

    R = dict(fresh=torch.tensor(rec["fresh"]), comm=torch.tensor(rec["comm"]), alive=torch.tensor(rec["alive"]),
             t_ep=torch.tensor(rec["t_ep"]), action=torch.tensor(rec["action"]),
             alive_post=torch.tensor(rec["alive_post"]), obs=obs_fn)
    tadv, tret = torch.tensor(adv), torch.tensor(ret)
    # checkpoints of (h, c) at the window starts, like the trainer records them during the rollout
    h = torch.zeros(B * N, H, dtype=torch.float64)
    c = torch.zeros_like(h)
    cks = []
    for t in range(T):
        if t % W == 0:
            cks.append((h.clone(), c.clone()))
        h, c, _ = bptt._forward(P, spec, R, t, h, c)
    dh = dc = None
    tot = dict(action_loss=0.0, value_loss=0.0, entropy=0.0)
    for k in reversed(range(len(cks))):
        t0, t1 = k * W, min(T, (k + 1) * W)
        dh, dc, st = bptt.window_backward(P, G, spec, R, t0, t1, cks[k][0], cks[k][1], tadv, tret, dh, dc)
        for q in tot:
            tot[q] += st[q]
    return G, tot


@pytest.mark.parametrize("name", golden_names("grad_"))
def test_manual_backward_matches_autograd_oracle(name):
    meta, _ = load_golden(name)
    T = 2 * meta["args"]["max_steps"] + 7                      # the last episode of every slot is cut by the batch end
    meta, args, p, rec, adv, ret, want, wstat = _lockstep_records(name, B=3, T=T)
    for W in (16, T):                                          # several chained windows, and one window
        G, tot = _run_manual(args, meta, p, rec, adv, ret, W)
        for q in wstat:
            assert np.isclose(tot[q], wstat[q], rtol=1e-9, atol=1e-9), (q, W)
        for key, v in want.items():
            if v is None:
                assert float(G[key].abs().max()) == 0.0, key   # hidd_encoder: unused by the forward
            else:
                assert np.allclose(G[key].numpy(), v, rtol=1e-8, atol=1e-10), (key, W)


@pytest.mark.parametrize("name", golden_names("grad_"))
def test_one_step_windows_from_recorded_states_equal_one_window(name):
    """The float64 reference of the BPTT kernel tests (tests/bptt_ref.py) runs one-step windows, each started from the
    recorded state entering its step, with (dh, dc) chained from the step after.  Given the exact per-step states
    this is the same backward as one window over the whole batch (detach cuts, episode starts, chained gradients)."""
    from bptt_ref import chain_one_step
    meta, _ = load_golden(name)
    T = 2 * meta["args"]["max_steps"] + 7
    meta, args, p, rec, adv, ret, want, wstat = _lockstep_records(name, B=3, T=T)
    G1, tot1 = _run_manual(args, meta, p, rec, adv, ret, T)
    N, H = args.nagents, args.hid_size
    B = rec["fresh"].shape[1]
    P = {k: torch.tensor(v, dtype=torch.float64) for k, v in p.items()}
    G = {k: torch.zeros_like(v) for k, v in P.items()}
    spec = bptt.Spec(N, H, len(meta["heads"]), bool(args.hard_attn) and bool(args.commnet),
                     getattr(args, "comm_mode", "avg") == "avg", bool(args.comm_mask_zero), args.value_coeff, args.entr,
                     args.detach_gap, args.max_steps)
    tobs = torch.tensor(rec["obs"]).reshape(T, B * N, -1)
    R = dict(fresh=torch.tensor(rec["fresh"]), comm=torch.tensor(rec["comm"]), alive=torch.tensor(rec["alive"]),
             t_ep=torch.tensor(rec["t_ep"]), action=torch.tensor(rec["action"]),
             alive_post=torch.tensor(rec["alive_post"]), obs=lambda t: tobs[t])
    states = [(torch.zeros(B * N, H, dtype=torch.float64), torch.zeros(B * N, H, dtype=torch.float64))]
    for t in range(T - 1):              # the state entering every step, as the kernel trainer records it (rec_h, rec_c)
        h, c, _ = bptt._forward(P, spec, R, t, *states[-1])
        states.append((h, c))
    tot = chain_one_step(P, G, spec, R, lambda t: states[t], torch.tensor(adv), torch.tensor(ret))
    for q in tot:
        assert np.isclose(tot[q], tot1[q], rtol=1e-12, atol=1e-12), (q, tot[q], tot1[q])
    for key in G:
        scale = max(float(G1[key].abs().max()), 1e-300)
        assert float((G[key] - G1[key]).abs().max()) <= 1e-12 * scale, key


def test_sparse_observation_path_equals_dense():
    meta, args, p, rec, adv, ret, want, _ = _lockstep_records("grad_pp_easy_ic3net", B=2, T=25)
    Gd, _ = _run_manual(args, meta, p, rec, adv, ret, 10)
    Gs, _ = _run_manual(args, meta, p, rec, adv, ret, 10, sparse=True)
    for key in Gd:
        assert torch.allclose(Gd[key], Gs[key], rtol=1e-11, atol=1e-13), key


@pytest.mark.parametrize("enemy", [False, True])
@pytest.mark.parametrize("dim,vision,n", [(5, 0, 3), (4, 1, 2), (6, 2, 5), (20, 1, 10)])
def test_sparse_pp_observation_equals_oracle_observation(dim, vision, n, enemy):
    """Trainer._pp_sparse_obs (the (index, value) form of the predator-prey observation both gradient paths consume)
    scattered back to dense equals the oracle's observation, incl. stacked predators, prey under a predator and
    windows that leave the grid.  Runs on CPU: the method only touches torch ops and four env attributes."""
    from types import SimpleNamespace
    from oracle.pp_env import PredatorPreyOracle
    from ic3net_b200.trainer import Trainer
    orc = PredatorPreyOracle(n, dim, vision, enemy_comm=enemy)      # enemy_comm: the prey's own row comes last
    na = n + int(enemy)
    rs = np.random.RandomState(dim * 10 + vision)
    B = 6
    loc = rs.randint(0, dim, size=(B, n + 1, 2))
    loc[0, 1] = loc[0, 0]                      # two predators on one cell
    loc[1, n] = loc[1, 0]                      # prey under a predator
    loc[2, 0] = (0, 0)                         # window leaves the grid (vision > 0)
    loc[3, :] = (dim - 1, dim - 1)             # everybody in one corner
    fake = SimpleNamespace(env=SimpleNamespace(env=SimpleNamespace(dim=dim, vision=vision, npredator=n,
                                                                   nagent_rows=na, vocab_size=orc.vocab_size)))
    idx, val = Trainer._pp_sparse_obs(fake, torch.tensor(loc, dtype=torch.int32))
    O = orc.obs_dim
    dense = torch.zeros(B * na, O, dtype=torch.float64)
    dense.scatter_add_(1, idx, val.double())
    for b in range(B):
        orc.reset(locs=loc[b])
        assert np.array_equal(dense[b * na:(b + 1) * na].numpy(), orc.flat_obs()), b
    # and through the encoder of bptt.py: sparse form == dense form
    P = {"encoder.weight": torch.randn(7, O, dtype=torch.float64), "encoder.bias": torch.randn(7, dtype=torch.float64)}
    assert torch.allclose(bptt.encode(P, (idx, val.double())), bptt.encode(P, dense), rtol=1e-12, atol=1e-12)
