"""The float64 oracle of the non-recurrent tanh policies (tests/ff_oracle.py: models.MLP and CommNet / IC3Net without
--recurrent) against the gradients of the UNMODIFIED reference's Trainer.run_batch + compute_grad
(tests/golden/gradff_*.npz, written by scripts/gen_golden_ff.py).  CPU only."""
import numpy as np
import pytest

from ff_oracle import ff_oracle, make_weights
from helpers import golden_names, load_golden, make_oracle_env, ns, tj_tables

NAMES = golden_names("gradff_")


def test_fixtures_present():
    assert NAMES == ["gradff_pp_hard_ic3net", "gradff_pp_ic3net_p2", "gradff_pp_mlp",
                     "gradff_tj_commnet_sum_share_p3"], NAMES


def model_of(meta):
    return "commnet" if meta["args"]["commnet"] else "mlp"


def oracle_weights(meta):
    from oracle import policy
    a = meta["args"]
    return policy.params_to_f64(make_weights(meta["weights_seed"], meta["obs_dim"], a["hid_size"], meta["heads"],
                                             a.get("comm_init", "uniform"), model_of(meta), int(a["comm_passes"]),
                                             bool(a["share_weights"])))


def replay(meta, z):
    from oracle import grad as ograd
    from oracle.rollout import run_episode
    args = ns(meta["args"])
    is_tj = args.env_name == "traffic_junction"
    p = oracle_weights(meta)
    env = make_oracle_env(args, tj_tables(z) if is_tj else None)
    with ff_oracle(model_of(meta), int(args.comm_passes), bool(args.share_weights)):
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
def test_gradient_golden_ff(name):
    meta, z = load_golden(name)
    args = ns(meta["args"])
    assert not args.recurrent
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
    P = int(args.comm_passes)
    heads = {"value_head.weight", "value_head.bias"} | {"heads.%d.%s" % (m, k) for m in range(len(meta["heads"]))
                                                       for k in ("weight", "bias")}
    if model_of(meta) == "mlp":
        want = heads | {"affine1.weight", "affine1.bias", "affine2.weight", "affine2.bias"}
    elif args.share_weights:
        want = heads | {"encoder.weight", "encoder.bias", "f_module.weight", "f_module.bias", "C_module.weight",
                        "C_module.bias"}
    else:
        want = heads | {"encoder.weight", "encoder.bias"} | {"%s.%d.%s" % (m, i, k) for m in ("f_modules", "C_modules")
                                                            for i in range(P) for k in ("weight", "bias")}
    assert checked == want, sorted(checked ^ want)
    # what each fixture exercises
    if name == "gradff_pp_mlp":
        assert len(eps) > 1 and args.entr > 0 and args.vision == 1
    if name == "gradff_pp_ic3net_p2":
        assert P == 2 and args.hard_attn
        comm = np.concatenate([ep["comm_in"] for ep in eps])
        assert comm.any() and not comm.all()                                 # real gates: some talk, some do not
    if name == "gradff_tj_commnet_sum_share_p3":
        assert P == 3 and args.share_weights and args.comm_mode == "sum"
        alive = np.concatenate([ep["alive"] for ep in eps])
        assert np.any(np.diff(alive, axis=0) > 0) and np.any(np.diff(alive, axis=0) < 0)   # cars spawn and leave
    if name == "gradff_pp_hard_ic3net":
        assert (args.nagents, args.dim, args.vision) == (10, 20, 1)
