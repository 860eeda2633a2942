"""The float64 tanh-RNN oracle (tests/rnn_oracle.py: the IC / IRIC baselines, models.RNN with rnn_type 'MLP') against
the gradients of the UNMODIFIED reference's Trainer.run_batch + compute_grad (tests/golden/gradrnn_*.npz, written by
scripts/gen_golden_rnn.py).  CPU only."""
import numpy as np
import pytest

from helpers import golden_names, load_golden, make_oracle_env, ns, tj_tables
from rnn_oracle import make_weights, rnn_oracle

NAMES = golden_names("gradrnn_")


def test_fixtures_present():
    assert NAMES == ["gradrnn_pp_hard_ic", "gradrnn_pp_ic_detach", "gradrnn_tj_iric"], NAMES


def replay(meta, z):
    """The oracle's episodes of the fixture's slot and its gradient: (episodes, grads, stat, extra)."""
    from oracle import grad as ograd
    from oracle import policy
    from oracle.rollout import run_episode
    args = ns(meta["args"])
    is_tj = args.env_name == "traffic_junction"
    p = policy.params_to_f64(make_weights(meta["weights_seed"], meta["obs_dim"], args.hid_size, meta["heads"]))
    env = make_oracle_env(args, tj_tables(z) if is_tj else None)
    with rnn_oracle():
        eps, tick, k = [], 0, 0
        while tick < meta["num_steps"]:
            ep = run_episode(env, p, args, meta["seed"], meta["env_id"], epoch=0, tick0=tick, episode=k)
            eps.append(ep)
            tick += ep["num_steps"]
            k += 1
        g, st, extra = ograd.compute_grad(p, eps, args)
    assert k == meta["num_episodes"]
    return eps, g, st, extra


@pytest.mark.parametrize("name", NAMES)
def test_gradient_golden_rnn(name):
    meta, z = load_golden(name)
    args = ns(meta["args"])
    assert args.rnn_type == "MLP" and not args.commnet and args.recurrent
    eps, g, st, extra = replay(meta, z)
    for q in ("action_loss", "value_loss", "entropy"):
        assert np.isclose(st[q], meta[q], rtol=1e-9, atol=1e-9), (q, st[q], meta[q])
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
    assert checked == {"affine1.weight", "affine1.bias", "affine2.weight", "affine2.bias", "value_head.weight",
                       "value_head.bias", "heads.0.weight", "heads.0.bias"}, checked
    # what each fixture exercises
    if name == "gradrnn_pp_ic_detach":
        assert len(eps) > 1 and any(ep["num_steps"] >= args.detach_gap for ep in eps)       # restarts and cuts
    if name == "gradrnn_tj_iric":
        assert args.mean_ratio == 0.0
        alive = np.concatenate([ep["alive"] for ep in eps])
        assert np.any(np.diff(alive, axis=0) > 0) and np.any(np.diff(alive, axis=0) < 0)   # cars spawn and leave
    if name == "gradrnn_pp_hard_ic":
        assert (args.nagents, args.dim, args.vision) == (10, 20, 1)
