"""CPU tests: the oracle's greedy mode (tests/greedy_oracle.py) against the tests/golden/greedy_* fixtures, which the
unmodified reference's Trainer.get_episode wrote with argmax actions (scripts/gen_golden_greedy.py)."""
import numpy as np
import pytest

from greedy_oracle import argmax_actions, greedy
from helpers import golden_names, load_golden, make_oracle_env, ns, tj_tables
from oracle import policy
from oracle.gen_golden import make_weights
from oracle.rollout import run_episode

NAMES = golden_names("greedy_")


def test_fixtures_cover_the_cases():
    assert NAMES == ["greedy_pp_enemy_ic3net", "greedy_pp_mixed_ic3net", "greedy_tj_medium_ic3net"]
    meta, z = load_golden("greedy_pp_mixed_ic3net")
    assert any(len(z["e%d_act" % i]) < meta["args"]["max_steps"] for i in range(len(meta["env_ids"])))  # early end
    meta, z = load_golden("greedy_tj_medium_ic3net")
    assert z["e0_alive"].sum(-1).max() > 0                                                        # cars spawn


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_greedy_episode(name):
    meta, z = load_golden(name)
    args = ns(meta["args"])
    is_tj = args.env_name == "traffic_junction"
    p = policy.params_to_f64(make_weights(meta["weights_seed"], meta["obs_dim"], args.hid_size, meta["heads"],
                                          args.comm_init))
    for i, env_id in enumerate(meta["env_ids"]):
        env = make_oracle_env(args, tj_tables(z) if is_tj else None)
        with greedy():
            ep = run_episode(env, p, args, meta["seed"], env_id, epoch=meta["epoch"])
        g = lambda k: z["e%d_%s" % (i, k)]
        assert np.array_equal(ep["act"], g("act"))
        assert np.array_equal(ep["reward"], g("reward"))
        assert np.array_equal(ep["alive"], g("alive"))
        assert np.array_equal(ep["emask"], g("emask")) and np.array_equal(ep["mini"], g("mini"))
        assert np.allclose(ep["value"], g("value"), rtol=1e-12, atol=1e-13)
        for k in range(len(meta["heads"])):
            assert np.allclose(ep["logp"][:, :, sum(meta["heads"][:k]):sum(meta["heads"][:k + 1])], g("logp%d" % k),
                               rtol=1e-12, atol=1e-13)
        assert ep["success"] == int(g("success"))


def test_argmax_takes_the_lowest_tied_index():
    act, margin = argmax_actions([np.array([[0.5, 0.5, 0.1], [0.1, 0.7, 0.7]]), np.array([[1.0], [2.0]])])
    assert act.tolist() == [[0, 0], [1, 0]] and margin[:, 0].tolist() == [0.0, 0.0]
