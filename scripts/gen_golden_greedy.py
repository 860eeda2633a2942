"""Write the tests/golden/greedy_*.npz fixtures: whole episodes of the UNMODIFIED reference's Trainer.get_episode
(trainer.py:26-126) with greedy actions.  The script replaces the reference's select_action (action_utils.py:27-36, as
trainer.py binds it) by the argmax of every head's float64 log-probs (the lowest index on a tie, torch.argmax); the
reference itself is not changed.  The environments' draws are routed to the Philox streams (oracle.gen_golden.RefRandom).
Each episode is replayed by the float64 oracle in its greedy mode (tests/greedy_oracle.py) before anything is written:
observations, actions, rewards and masks exactly, hidden states and values to 1e-12 (oracle.gen_golden
.gen_episode_case).

    IC3NET_REFERENCE=<reference checkout> python scripts/gen_golden_greedy.py"""
import os
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

CASES = [
    # predator-prey IC3Net, mixed mode on a small board: episodes end early when every predator reaches the prey
    ("greedy_pp_mixed_ic3net", 101, (0, 1, 2, 3), 116, (0, 1, 5), dict(env_name="predator_prey", nagents=3, dim=3,
                                                                     vision=0, max_steps=20, hid_size=128,
                                                                     ic3net=True)),
    # predator-prey --enemy_comm: the prey is one more agent row of the policy
    ("greedy_pp_enemy_ic3net", 102, (0, 3), 112, (0, 1, 8), dict(env_name="predator_prey", nagents=3, dim=5, vision=0,
                                                                 max_steps=15, hid_size=128, ic3net=True,
                                                                 enemy_comm=True, nenemies=1)),
    # traffic-junction IC3Net, medium: cars spawn, move and complete their routes
    ("greedy_tj_medium_ic3net", 103, (0, 5), 113, (0, 1, 20), dict(env_name="traffic_junction", nagents=10, dim=14,
                                                                    vision=0, max_steps=40, hid_size=128, ic3net=True,
                                                                    difficulty="medium", add_rate_min=0.3,
                                                                    add_rate_max=0.3)),
]


def greedy_select(args, action_out):
    """select_action (action_utils.py:27-36) with the multinomial draw replaced by the argmax; same shapes."""
    import torch
    return torch.stack([torch.stack([z.argmax(-1, keepdim=True).detach() for z in x]) for x in action_out])


def main():
    warnings.filterwarnings("ignore")
    from oracle import gen_golden, ref_shims
    import greedy_oracle
    ref_shims.install()
    import trainer as ref_trainer
    ref_trainer.select_action = greedy_select
    with greedy_oracle.greedy():
        for name, seed, env_ids, wseed, hsteps, kw in CASES:
            gen_golden.gen_episode_case(name, seed, env_ids, wseed, hsteps=hsteps, **kw)
            print("wrote", name)


if __name__ == "__main__":
    main()
