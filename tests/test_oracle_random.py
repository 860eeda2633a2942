"""The Random baseline (models.Random) on CPU: the float64 oracle of tests/random_oracle.py against whole batches of the
UNMODIFIED reference's Trainer.run_batch + compute_grad (tests/golden/random_*.npz, written by
scripts/gen_golden_random.py), the host-side argument checks of ic3_random_policy_step, and the refusal of
--random --recurrent."""
import argparse
import ctypes

import numpy as np
import pytest

from helpers import golden_names, load_golden, make_oracle_env, ns, tj_tables
from random_oracle import losses, run_batch

NAMES = golden_names("random_")


def test_fixtures_present():
    assert NAMES == ["random_pp_enemy", "random_pp_small", "random_tj_medium"], NAMES


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_reference_batch(name):
    meta, z = load_golden(name)
    args = ns(meta["args"])
    args.naction_heads = meta["heads"]
    is_tj = args.env_name == "traffic_junction"
    eps = run_batch(make_oracle_env(args, tj_tables(z) if is_tj else None), args, meta["seed"], meta["env_id"])
    assert len(eps) == meta["num_episodes"] and sum(ep["num_steps"] for ep in eps) == meta["num_steps"]
    got = {k: np.concatenate([ep[k] for ep in eps]) for k in ("act", "loc", "reward", "emask", "mini", "alive",
                                                              "value", "logp")}
    for k in ("act", "loc", "reward", "emask", "mini", "alive"):
        assert np.array_equal(got[k], z[k]), k                 # actions and env state bit-exact
    for k in ("value", "logp"):
        assert np.allclose(got[k], z[k], rtol=0, atol=1e-12), k
    if meta["success"] >= 0:
        assert sum(ep["success"] for ep in eps) == meta["success"]
    st, ret = losses(eps, args)
    assert np.allclose(ret, z["returns"], rtol=0, atol=1e-12)
    for q in ("action_loss", "value_loss", "entropy"):
        assert np.isclose(st[q], meta[q], rtol=1e-8, atol=1e-8), (q, st[q], meta[q])
    # what each fixture exercises
    if name == "random_tj_medium":
        d = np.diff(z["alive"], axis=0)
        assert (d > 0).any() and (d < 0).any()                 # cars spawn and leave
        assert args.normalize_rewards and args.entr > 0
    if name == "random_pp_enemy":
        assert args.enemy_comm and z["act"].shape[1] == args.nfriendly + 1


def test_random_policy_step_validates_arguments_before_touching_the_device(built_lib):
    """Bad calls return IC3_E_NULL / IC3_E_RANGE from the host-side checks; nothing is launched, so no GPU is needed."""
    from ic3net_b200 import _lib
    lib = _lib.load()
    E_NULL, E_RANGE = -1, -2
    fake = 0x1000                      # never dereferenced: validation fails first

    def cfg(heads=(5,), **kw):
        hd = (ctypes.c_int32 * _lib.MAX_HEADS)(*heads)
        return _lib.PolicyCfg(**dict(dict(B=4, N=3, nheads=len(heads), head_dim=hd, env_id0=0, seed=1), **kw))

    io = _lib.PolicyIO(value=fake, logp=fake, action=fake)
    call = lambda c, i=io: lib.ic3_random_policy_step(ctypes.byref(c) if c is not None else None,
                                                      ctypes.byref(i) if i is not None else None, None, None)
    assert call(None) == E_NULL and call(cfg(), None) == E_NULL
    assert call(cfg(), _lib.PolicyIO(logp=fake)) == E_NULL and call(cfg(), _lib.PolicyIO(value=fake)) == E_NULL
    for bad in (dict(B=0), dict(N=0), dict(N=_lib.MAX_AGENTS + 1), dict(nheads=0), dict(nheads=_lib.MAX_HEADS + 1)):
        assert call(cfg(**bad)) == E_RANGE, bad
    for heads in ((0,), (_lib.MAX_HEAD_DIM + 1,), (5, 3), (2, 2, 2, 2)):    # empty / wide heads, > 7 logits
        assert call(cfg(heads)) == E_RANGE, heads


def test_random_recurrent_is_refused():
    """--random --recurrent fails in the reference (Random.forward gets [state, prev_hid]); Trainer refuses it up front,
    before it touches the policy, the environment or the device."""
    from ic3net_b200.models import Random
    from ic3net_b200.trainer import Trainer
    net = Random.__new__(Random)       # the check needs the type alone; building one needs a GPU
    with pytest.raises(ValueError, match="not recurrent"):
        Trainer(argparse.Namespace(recurrent=True), net, None)
