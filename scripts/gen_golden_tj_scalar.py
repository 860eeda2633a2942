"""Write the tests/golden/tj_scalar_*.npz fixtures: the traffic junction with ``--vocab_type scalar`` as the UNMODIFIED
reference builds and runs it, through oracle/gen_golden.py's case writers inside the scalar-vocabulary oracle context of
tests/tj_scalar_oracle.py -- so a trajectory, episode or gradient fixture is written only after the oracle replay has
matched the reference (observations bit for bit, float64 policy outputs to 1e-11, every gradient to 1e-8).

  tj_scalar_tables_<difficulty>_<dim>  the reference env's grid and routes, its classes and GymWrapper.observation_dim
                                       at vision 1
  tj_scalar_env_*                      env trajectories (random actions, cars spawning, crashing and leaving)
  tj_scalar_ep_*                       one IC3Net episode through the reference's Trainer.get_episode
  tj_scalar_grad_*                     one Trainer.run_batch + compute_grad at hid_size 128

    IC3NET_REFERENCE=<reference checkout> python scripts/gen_golden_tj_scalar.py"""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

TABLES = [("easy", 6), ("easy", 10), ("medium", 6), ("medium", 14), ("hard", 9), ("hard", 18)]
TJ = dict(env_name="traffic_junction", vocab_type="scalar")
ENV_CASES = [
    ("tj_scalar_env_easy", 40, 26, 0, dict(TJ, nagents=5, dim=6, vision=0, difficulty="easy", add_rate_min=0.3,
                                           add_rate_max=0.3)),
    ("tj_scalar_env_medium_v1", 40, 27, 2, dict(TJ, nagents=10, dim=14, vision=1, difficulty="medium",
                                                add_rate_min=0.3, add_rate_max=0.3)),
    ("tj_scalar_env_hard", 50, 28, 3, dict(TJ, nagents=20, dim=18, vision=0, difficulty="hard", add_rate_min=0.25,
                                           add_rate_max=0.25)),
]


def gen_tables():
    from oracle import gen_golden, ref_shims
    from tj_scalar_oracle import CAR, OUTSIDE, VOCAB
    for diff, dim in TABLES:
        a = ref_shims.make_args(nagents=4, dim=dim, vision=1, difficulty=diff, ic3net=True, **TJ)
        w = ref_shims.make_ref_env(a)
        env = w.env
        assert env.OUTSIDE_CLASS == OUTSIDE and env.CAR_CLASS == CAR and env.vocab_size == VOCAB
        assert not hasattr(env, "BASE")
        t = gen_golden.tj_tables_from_ref(env)
        ln, cells = gen_golden.pack_routes(t["routes"])
        gen_golden.save("tj_scalar_tables_%s_%d" % (diff, dim),
                        dict(difficulty=diff, dim=dim, vision=1, dims=list(map(int, env.dims)), OUTSIDE=OUTSIDE,
                             CAR=CAR, vocab=VOCAB, npath=int(env.npath), obs_dim=int(w.observation_dim)),
                        grid=t["grid"], route_len=ln, route_cells=cells)


def main():
    warnings.filterwarnings("ignore")
    from oracle import gen_golden
    from tj_scalar_oracle import scalar_oracle
    np.seterr(all="ignore")
    gen_tables()
    with scalar_oracle():
        for name, T, seed, env_id, kw in ENV_CASES:
            gen_golden.gen_env_case(name, T, seed, env_id, **kw)
        gen_golden.gen_episode_case("tj_scalar_ep_medium_ic3net", 48, (0, 3), 58, hsteps=(0, 1, 20), nagents=10,
                                    dim=14, vision=1, max_steps=40, hid_size=128, ic3net=True, difficulty="medium",
                                    add_rate_min=0.2, add_rate_max=0.2, **TJ)
        gen_golden.gen_grad_case("tj_scalar_grad_hard_ic3net_h128", 72, 5, 82, nagents=20, dim=18, vision=0,
                                 max_steps=25, hid_size=128, ic3net=True, difficulty="hard", add_rate_min=0.2,
                                 add_rate_max=0.2, batch_size=40, detach_gap=10, **TJ)
    return 0


if __name__ == "__main__":
    sys.exit(main())
