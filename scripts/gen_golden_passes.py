"""Write the tests/golden/gradpasses_*.npz fixtures: the gradient of a whole batch through the UNMODIFIED reference's
Trainer.run_batch + compute_grad for CommNet / IC3Net with comm_passes > 1 (and share_weights), by
oracle.gen_golden.gen_grad_case inside the multi-pass oracle context of tests/passes_oracle.py -- so the fixture is
written only after the float64 oracle replay has matched the reference (loss sums to 1e-9, every gradient to 1e-8).

    IC3NET_REFERENCE=<reference checkout> python scripts/gen_golden_passes.py"""
import os
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

CASES = [
    # IC3Net, predator-prey hard geometry, two passes, detach_gap cuts
    ("gradpasses_pp_hard_ic3net_p2", 72, 4, 82, dict(env_name="predator_prey", nagents=10, dim=20, vision=1,
     max_steps=20, hid_size=128, ic3net=True, batch_size=35, detach_gap=8, comm_passes=2)),
    # CommNet (soft attention), traffic junction, three passes of one shared C module, summed messages
    ("gradpasses_tj_easy_commnet_sum_share_p3", 73, 1, 83, dict(env_name="traffic_junction", nagents=5, dim=6,
     vision=0, max_steps=20, hid_size=128, commnet=True, comm_mode="sum", difficulty="easy", add_rate_min=0.3,
     add_rate_max=0.3, batch_size=50, mean_ratio=0.5, gamma=0.9, entr=0.005, comm_passes=3, share_weights=True)),
    # IC3Net with --enemy_comm (the prey talks), four passes
    ("gradpasses_pp_enemy_ic3net_p4", 74, 5, 84, dict(env_name="predator_prey", nagents=3, dim=5, vision=1,
     max_steps=12, hid_size=128, ic3net=True, enemy_comm=True, batch_size=40, detach_gap=5, comm_passes=4)),
]


def main():
    warnings.filterwarnings("ignore")
    from oracle import gen_golden
    from passes_oracle import passes_oracle
    for name, seed, env_id, wseed, kw in CASES:
        with passes_oracle(kw["comm_passes"], kw.get("share_weights", False)):
            gen_golden.gen_grad_case(name, seed, env_id, wseed, **kw)
        print("wrote", name, flush=True)


if __name__ == "__main__":
    main()
