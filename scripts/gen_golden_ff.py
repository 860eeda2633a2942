"""Write the tests/golden/gradff_*.npz fixtures: the gradient of a whole batch through the UNMODIFIED reference's
Trainer.run_batch + compute_grad for the non-recurrent tanh policies -- models.MLP (what the reference's main.py builds
when no model flag is given) and CommNet / IC3Net without --recurrent -- by oracle.gen_golden.gen_grad_case inside the
oracle context of tests/ff_oracle.py, so a fixture is written only after the float64 oracle replay has matched the
reference (loss sums to 1e-9, every gradient to 1e-8).

For models.MLP, gen_grad_case's policy (which it imports as the reference's comm.CommNetMLP) is bound to the reference's
own models.MLP for the duration of the case (in memory only: the reference files are not touched).

    IC3NET_REFERENCE=<reference checkout> python scripts/gen_golden_ff.py"""
import contextlib
import os
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

NONREC = dict(recurrent=False, rnn_type="MLP", hid_size=128)
CASES = [
    # models.MLP, predator-prey with vision 1, short episodes inside the batch, entropy bonus
    ("gradff_pp_mlp", "mlp", 91, 2, 101, dict(NONREC, commnet=False, ic3net=False, hard_attn=False,
     env_name="predator_prey", nagents=3, dim=5, vision=1, max_steps=12, batch_size=40, entr=0.01)),
    # non-recurrent IC3Net, predator-prey, hard-attention gates that switch, two passes
    ("gradff_pp_ic3net_p2", "commnet", 92, 3, 102, dict(NONREC, commnet=True, ic3net=False, hard_attn=True,
     env_name="predator_prey", nagents=4, dim=6, vision=1, max_steps=15, batch_size=40, comm_passes=2)),
    # non-recurrent CommNet, traffic junction with cars spawning and leaving, three shared passes, summed messages
    ("gradff_tj_commnet_sum_share_p3", "commnet", 93, 1, 103, dict(NONREC, commnet=True, ic3net=False,
     hard_attn=False, env_name="traffic_junction", nagents=5, dim=6, vision=0, max_steps=20, difficulty="easy",
     add_rate_min=0.3, add_rate_max=0.3, batch_size=50, mean_ratio=0.5, gamma=0.9, comm_mode="sum", comm_passes=3,
     share_weights=True)),
    # non-recurrent IC3Net, the predator-prey hard geometry (10 agents, dim 20, vision 1)
    ("gradff_pp_hard_ic3net", "commnet", 94, 4, 104, dict(NONREC, commnet=True, ic3net=False, hard_attn=True,
     env_name="predator_prey", nagents=10, dim=20, vision=1, max_steps=20, batch_size=35)),
]


@contextlib.contextmanager
def reference_policy(model):
    from oracle import ref_shims
    ref_shims.install()
    import comm
    import models
    saved = comm.CommNetMLP
    if model == "mlp":
        comm.CommNetMLP = models.MLP
    try:
        yield
    finally:
        comm.CommNetMLP = saved


def main():
    warnings.filterwarnings("ignore")
    from oracle import gen_golden
    from ff_oracle import ff_oracle
    only = sys.argv[1:]
    for name, model, seed, env_id, wseed, kw in CASES:
        if only and name not in only:
            continue
        with reference_policy(model), ff_oracle(model, kw.get("comm_passes", 1), kw.get("share_weights", False)):
            gen_golden.gen_grad_case(name, seed, env_id, wseed, **kw)
        print("wrote", name, flush=True)


if __name__ == "__main__":
    main()
