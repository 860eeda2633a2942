"""Write the tests/golden/random_*.npz fixtures: whole batches of the UNMODIFIED reference's Trainer.run_batch +
compute_grad with models.Random (main.py:166-167, models.py:37-56).  The reference's draws are routed to the Philox
streams: the environments' and torch.multinomial's by oracle.gen_golden.RefRandom, and torch.rand / torch.randn inside
Random.forward to stream 4 (tests/random_oracle.py), for the duration of each forward call only.  A fixture is written
only after the float64 oracle of tests/random_oracle.py has replayed the batch: actions, env state, rewards and masks
exactly, values and log-probs to 1e-12, loss sums to 1e-9.  The reference's optimizer step after compute_grad is
checked to leave the parameter and the RMSprop state untouched (no gradient reaches the parameter).

    IC3NET_REFERENCE=<reference checkout> python scripts/gen_golden_random.py"""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

RANDOM = dict(random=True, commnet=False, ic3net=False, hard_attn=False, recurrent=False)
CASES = [
    # predator-prey on a small board (mixed mode: an episode ends early when every predator reaches the prey)
    ("random_pp_small", 90, 2, dict(RANDOM, env_name="predator_prey", nagents=3, dim=4, vision=1, max_steps=15,
                                     batch_size=40)),
    # traffic junction medium: cars spawn, complete their routes and leave; discounted, normalised, entropy term
    ("random_tj_medium", 91, 1, dict(RANDOM, env_name="traffic_junction", nagents=10, dim=14, vision=1, max_steps=40,
                                      difficulty="medium", add_rate_min=0.3, add_rate_max=0.3, batch_size=80,
                                      gamma=0.9, normalize_rewards=True, entr=0.01)),
    # predator-prey --enemy_comm: the prey is one more agent row of the policy
    ("random_pp_enemy", 92, 3, dict(RANDOM, env_name="predator_prey", nagents=3, dim=4, vision=0, max_steps=12,
                                     enemy_comm=True, batch_size=30, mean_ratio=0.5)),
]


class Stream4(object):
    """torch.rand / torch.randn of Random.forward (models.py:47-54) on Philox stream 4 at the env's current tick."""

    def __init__(self, rr, heads):
        self.rr, self.heads = rr, list(heads)

    def rand(self, size, **kw):
        import torch
        import random_oracle
        _, n, one = tuple(size)
        assert one == 1
        self.u = random_oracle.words(self.rr.seed, self.rr.env_id, self.rr.tick, np.arange(n))
        self.k = 0
        return torch.tensor(self.u[:, 0] * 2.0 ** -24).view(1, n, 1)

    def randn(self, size, **kw):
        import torch
        import random_oracle
        _, n, na = tuple(size)
        assert na == self.heads[self.k]
        off = sum(self.heads[:self.k])
        z = random_oracle.value_logits(self.u, sum(self.heads))[1][:, off:off + na]
        self.k += 1
        return torch.tensor(z).view(1, n, na)


def gen_case(name, seed, env_id, kw):
    import torch
    import random_oracle
    from oracle import gen_golden, ref_shims
    torch.set_default_dtype(torch.float64)
    ref_shims.install()
    from models import Random
    from trainer import Trainer
    args = ref_shims.make_args(**kw)
    w = ref_shims.make_ref_env(args)
    ref_shims.finish_args(args, w)
    net = Random(args, args.num_inputs)
    param0 = net.parameter.detach().clone()
    tr = Trainer(args, net, w)
    is_tj = args.env_name == "traffic_junction"
    tables = gen_golden.tj_tables_from_ref(w.env) if is_tj else None
    rr = gen_golden.RefRandom(seed, env_id)
    s4 = Stream4(rr, args.naction_heads)
    orig_step, orig_reset, orig_fwd = w.step, w.reset, net.forward
    locs = []

    def step(action, _o=orig_step):
        rr.group = -1
        out = _o(action)
        rr.tick += 1
        rr.head = 0
        e = w.env
        locs.append(np.array(e.car_loc) if is_tj else np.concatenate([e.predator_loc, e.prey_loc]))
        return out

    def reset(epoch, _o=orig_reset):
        out = _o(epoch)
        rr.episode += 1
        return out

    def forward(x, info={}, _o=orig_fwd):
        saved = torch.rand, torch.randn
        torch.rand, torch.randn = s4.rand, s4.randn
        try:
            return _o(x, info)
        finally:
            torch.rand, torch.randn = saved
    w.step, w.reset, net.forward = step, reset, forward
    with gen_golden.routed(rr):
        batch, stat = tr.run_batch(0)
    w.step, w.reset, net.forward = orig_step, orig_reset, orig_fwd
    tr.optimizer.zero_grad()
    s = tr.compute_grad(batch)
    assert net.parameter.grad is None
    tr.optimizer.step()                                     # trainer.py:251-254
    assert tr.optimizer.state_dict()["state"] == {} and torch.equal(net.parameter.detach(), param0)
    T, n = stat["num_steps"], args.nagents
    ref = dict(act=np.array(batch.action).transpose(0, 2, 1),
               value=torch.cat(batch.value).view(T, n).detach().numpy(),
               logp=np.stack([torch.cat(list(a), -1)[0].detach().numpy() for a in batch.action_out]),
               reward=np.array(batch.reward), emask=np.array(batch.episode_mask),
               mini=np.array(batch.episode_mini_mask),
               alive=np.array([m["alive_mask"] for m in batch.misc]), loc=np.array(locs))
    # ---- oracle replay ----
    eps = random_oracle.run_batch(gen_golden.make_oracle_env(args, tables), args, seed, env_id)
    orc = {k: np.concatenate([ep[k] for ep in eps]) for k in ref}
    assert len(eps) == stat["num_episodes"] and len(orc["act"]) == T
    for k in ("act", "reward", "emask", "mini", "alive", "loc"):
        assert np.array_equal(orc[k], ref[k]), (name, k)
    for k in ("value", "logp"):
        assert np.allclose(orc[k], ref[k], rtol=0, atol=1e-12), (name, k, np.abs(orc[k] - ref[k]).max())
    ol, ret = random_oracle.losses(eps, args)
    for q in ("action_loss", "value_loss", "entropy"):
        assert np.isclose(ol[q], s[q], rtol=1e-9, atol=1e-9), (name, q, ol[q], s[q])
    if "success" in stat:
        assert sum(ep["success"] for ep in eps) == stat["success"]
    meta = dict(kind="random", seed=seed, env_id=env_id,
                args={k_: v for k_, v in vars(args).items() if isinstance(v, (int, float, str, bool))},
                heads=list(map(int, args.naction_heads)), num_steps=int(T), num_episodes=int(stat["num_episodes"]),
                success=int(stat.get("success", -1)), action_loss=float(s["action_loss"]),
                value_loss=float(s["value_loss"]), entropy=float(s["entropy"]))
    arrays = dict(ref, returns=ret, margin=np.concatenate([ep["margin"] for ep in eps]))
    if is_tj:
        arrays["grid"] = tables["grid"]
        arrays["route_len"], arrays["route_cells"] = gen_golden.pack_routes(tables["routes"])
    gen_golden.save(name, meta, **arrays)


def main():
    warnings.filterwarnings("ignore")
    for name, seed, env_id, kw in CASES:
        gen_case(name, seed, env_id, kw)


if __name__ == "__main__":
    main()
