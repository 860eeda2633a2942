"""The float64 multi-pass oracle (tests/passes_oracle.py) against the gradients of the UNMODIFIED reference's
Trainer.compute_grad with comm_passes > 1 and share_weights (tests/golden/gradpasses_*.npz, written by
scripts/gen_golden_passes.py).  CPU only."""
import numpy as np
import pytest

from helpers import golden_names, load_golden, make_oracle_env, ns, tj_tables
from passes_oracle import make_weights, passes_oracle

NAMES = golden_names("gradpasses_")


def test_fixtures_present():
    assert len(NAMES) == 3, NAMES


@pytest.mark.parametrize("name", NAMES)
def test_gradient_golden_passes(name):
    from oracle import grad as ograd
    from oracle import policy
    from oracle.rollout import run_episode
    meta, z = load_golden(name)
    args = ns(meta["args"])
    passes, share = int(args.comm_passes), bool(args.share_weights)
    assert passes > 1
    is_tj = args.env_name == "traffic_junction"
    sd = make_weights(meta["weights_seed"], meta["obs_dim"], args.hid_size, meta["heads"], args.comm_init, passes, share)
    p = policy.params_to_f64(sd)
    env = make_oracle_env(args, tj_tables(z) if is_tj else None)
    with passes_oracle(passes, share):
        eps, tick, k = [], 0, 0
        while tick < meta["num_steps"]:
            ep = run_episode(env, p, args, meta["seed"], meta["env_id"], epoch=0, tick0=tick, episode=k)
            eps.append(ep)
            tick += ep["num_steps"]
            k += 1
        g, st, extra = ograd.compute_grad(p, eps, args)
    assert k == meta["num_episodes"]
    assert np.isclose(st["action_loss"], meta["action_loss"], rtol=1e-9, atol=1e-9)
    assert np.isclose(st["value_loss"], meta["value_loss"], rtol=1e-9, atol=1e-9)
    assert np.isclose(st["entropy"], meta["entropy"], rtol=1e-9, atol=1e-9)
    assert np.allclose(extra["returns"], z["returns"], rtol=1e-12, atol=1e-12)
    checked = set()
    for key in z.files:
        if key.startswith("g_"):
            assert np.allclose(g[key[2:]], z[key], rtol=1e-8, atol=1e-10), key
            checked.add(key[2:])
        elif key.startswith("gsample_"):
            q = g[key[8:]]
            assert np.allclose(q.ravel()[::max(1, q.size // 2048)][:2048], z[key], rtol=1e-8, atol=1e-10), key
            assert np.allclose([q.sum(), np.abs(q).sum(), (q ** 2).sum()], z["gsum_" + key[8:]], rtol=1e-8)
            checked.add(key[8:])
    c_names = {k for k in checked if k.startswith("C_module")}
    assert c_names == ({"C_module.weight", "C_module.bias"} if share else
                       {"C_modules.%d.%s" % (i, w) for i in range(passes) for w in ("weight", "bias")}), c_names
    assert len(checked) >= 8
