"""Write the tests/golden/gradrnn_*.npz fixtures: the gradient of a whole batch through the UNMODIFIED reference's
Trainer.run_batch + compute_grad with models.RNN and the tanh recurrence (rnn_type 'MLP': the IC / IRIC baselines, as
main.py:168-169 builds them for --recurrent without --commnet), by oracle.gen_golden.gen_grad_case inside the tanh-RNN
oracle context of tests/rnn_oracle.py -- so a fixture is written only after the float64 oracle replay has matched the
reference (loss sums to 1e-9, every gradient to 1e-8).

gen_grad_case builds the policy the reference's comm module exports as CommNetMLP; for the duration of each case that
name is bound to the reference's own models.RNN (in memory only: the reference files are not touched).

The prefix is gradrnn_, not grad_: the grad_* fixtures are CommNet / IC3Net cases that several tests build as such.

    IC3NET_REFERENCE=<reference checkout> python scripts/gen_golden_rnn.py"""
import contextlib
import os
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

IC = dict(commnet=False, ic3net=False, hard_attn=False, recurrent=True, rnn_type="MLP", hid_size=128)
CASES = [
    # IC, predator-prey with vision 1, short episodes inside the batch and detach_gap cuts
    ("gradrnn_pp_ic_detach", 75, 2, 85, dict(IC, env_name="predator_prey", nagents=3, dim=5, vision=1, max_steps=12,
     batch_size=40, detach_gap=5, entr=0.01)),
    # IRIC (mean_ratio 0), traffic junction: cars spawn, complete their routes and leave (alive changes per step)
    ("gradrnn_tj_iric", 76, 1, 86, dict(IC, env_name="traffic_junction", nagents=5, dim=6, vision=0, max_steps=20,
     difficulty="easy", add_rate_min=0.3, add_rate_max=0.3, batch_size=50, mean_ratio=0.0, gamma=0.9,
     normalize_rewards=True)),
    # IC, the predator-prey hard geometry (10 agents, dim 20, vision 1)
    ("gradrnn_pp_hard_ic", 77, 4, 87, dict(IC, env_name="predator_prey", nagents=10, dim=20, vision=1, max_steps=20,
     batch_size=35, detach_gap=8)),
]


@contextlib.contextmanager
def reference_rnn_policy():
    """gen_grad_case's policy is the reference's models.RNN (it imports the class as comm.CommNetMLP)."""
    from oracle import ref_shims
    ref_shims.install()
    import comm
    import models
    saved = comm.CommNetMLP
    comm.CommNetMLP = models.RNN
    try:
        yield
    finally:
        comm.CommNetMLP = saved


def main():
    warnings.filterwarnings("ignore")
    from oracle import gen_golden
    from rnn_oracle import rnn_oracle
    for name, seed, env_id, wseed, kw in CASES:
        with reference_rnn_policy(), rnn_oracle():
            gen_golden.gen_grad_case(name, seed, env_id, wseed, **kw)
        print("wrote", name, flush=True)


if __name__ == "__main__":
    main()
