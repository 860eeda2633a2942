"""CPU tests of the traffic junction with ``vocab_type='scalar'``: the host tables and the CPU oracle against the fixtures
written from the unmodified reference (scripts/gen_golden_tj_scalar.py), the ic3_tj_cfg layout, the argument checks of
the TJ entry points, and the gradient kernels' coverage, which excludes this vocabulary.  No device work."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from helpers import golden_names, load_golden, ns, tj_tables
from oracle import policy
from oracle.gen_golden import make_weights
from tj_scalar_oracle import CAR, OUTSIDE, VOCAB, make_env

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E_NULL, E_RANGE, E_UNSUPPORTED = -1, -2, -3


@pytest.mark.parametrize("name", golden_names("tj_scalar_tables_"))
def test_host_tables_match_the_reference(name):
    from ic3net_b200 import traffic_helper
    meta, z = load_golden(name)
    t = traffic_helper.build_tables(meta["difficulty"], meta["dim"], meta["vision"], "scalar")
    assert np.array_equal(t["grid"], z["grid"])
    assert set(np.unique(t["grid"])) == {0, 1}                 # road class only, no per-cell numbering
    assert (t["OUTSIDE"], t["CAR"], t["vocab"], t["BASE"]) == (OUTSIDE, CAR, VOCAB, None)
    assert tuple(t["dims"]) == tuple(meta["dims"]) and t["npath"] == meta["npath"]
    routes = tj_tables(z)["routes"]
    assert [len(g) for g in routes] == [len(g) for g in t["routes"]]
    for ga, gb in zip(routes, t["routes"]):
        for pa, pb in zip(ga, gb):
            assert np.array_equal(pa, pb)
    # the routes are the bool vocabulary's: both hand get_routes the road-class grid
    tb = traffic_helper.build_tables(meta["difficulty"], meta["dim"], meta["vision"], "bool")
    assert np.array_equal(tb["route_cells"], t["route_cells"]) and np.array_equal(tb["route_len"], t["route_len"])
    W = 2 * meta["vision"] + 1
    assert meta["obs_dim"] == 4 + W * W * 2                     # GymWrapper.observation_dim of the reference


def test_observation_dim_of_the_spaces():
    """observation_dim counts the MultiDiscrete(dims) position member as 2, whatever the easy +1 of dims."""
    from ic3net_b200 import spaces
    from ic3net_b200.env_wrappers import per_agent_obs_dim
    for dim, vision in ((6, 0), (14, 1), (18, 2)):
        W = 2 * vision + 1
        sp = spaces.Tuple((spaces.Discrete(2), spaces.Discrete(12), spaces.MultiDiscrete((dim, dim)),
                           spaces.MultiBinary((W, W, 2))))
        assert per_agent_obs_dim(sp, spaces.Discrete(2)) == 4 + W * W * 2


def test_float32_p_norm_equals_the_float64_division_rounded():
    """The kernels divide in float32; the reference divides in float64 and the observation reaches float32 once.  For
    every position of every board up to 64 cells the two agree, so the observations are bit-exact."""
    for d in range(1, 64):
        r = np.arange(d + 1)
        f32 = r.astype(np.float32) / np.float32(d)
        assert np.array_equal(f32, (r / d).astype(np.float32)), d


@pytest.mark.parametrize("name", golden_names("tj_scalar_env_"))
def test_oracle_env_trajectory(name):
    meta, z = load_golden(name)
    args = ns(meta["args"])
    assert args.vocab_type == "scalar"
    env = make_env(args, tj_tables(z))
    seed, env_id = meta["seed"], meta["env_id"]
    obs = env.reset(0)
    assert obs.shape[1] == meta["obs_dim"]
    assert np.array_equal(obs, z["obs0"]) and np.array_equal(env.car_loc, z["loc0"])
    for t in range(len(z["act"])):
        obs, r, done, info = env.step(z["act"][t], seed=seed, env_id=env_id)
        assert np.array_equal(info["alive_mask"], z["alive"][t])
        assert np.array_equal(info["is_completed"], z["completed"][t])
        assert np.array_equal(env.car_loc, z["loc"][t]), (name, t)
        assert np.array_equal(np.stack([env.wait, env.route_id, env.last_act, env.route_loc], 1), z["aux"][t])
        assert np.array_equal(r, z["reward"][t]), (name, t)
        assert np.array_equal(obs.astype(np.float32), z["obs"][t]), (name, t)
    # the trajectory covers spawning, crashes and cars leaving the map
    assert z["alive"].sum(1).max() >= 2 and z["completed"].sum() > 0 and (z["reward"] <= -10).any()


def test_oracle_episode():
    from oracle.rollout import run_episode
    meta, z = load_golden("tj_scalar_ep_medium_ic3net")
    args = ns(meta["args"])
    p = policy.params_to_f64(make_weights(meta["weights_seed"], meta["obs_dim"], args.hid_size, meta["heads"],
                                          args.comm_init))
    for i, env_id in enumerate(meta["env_ids"]):
        ep = run_episode(make_env(args, tj_tables(z)), p, args, meta["seed"], env_id, epoch=meta["epoch"])
        g = lambda k: z["e%d_%s" % (i, k)]
        assert np.array_equal(ep["act"], g("act")) and np.array_equal(ep["reward"], g("reward"))
        assert np.array_equal(ep["alive"], g("alive"))
        assert np.array_equal(ep["emask"], g("emask")) and np.array_equal(ep["mini"], g("mini"))
        assert np.allclose(ep["value"], g("value"), rtol=1e-12, atol=1e-13)
        for j, t in enumerate(g("h_steps")):
            assert np.allclose(ep["h"][t], g("h_sel")[j], rtol=1e-12, atol=1e-13)
            assert np.allclose(ep["c"][t], g("c_sel")[j], rtol=1e-12, atol=1e-13)


def test_oracle_gradient():
    from oracle import grad as ograd
    from oracle.rollout import run_episode
    meta, z = load_golden("tj_scalar_grad_hard_ic3net_h128")
    args = ns(meta["args"])
    p = policy.params_to_f64(make_weights(meta["weights_seed"], meta["obs_dim"], args.hid_size, meta["heads"],
                                          args.comm_init))
    env = make_env(args, tj_tables(z))
    eps, tick, k = [], 0, 0
    while tick < meta["num_steps"]:
        eps.append(run_episode(env, p, args, meta["seed"], meta["env_id"], epoch=0, tick0=tick, episode=k))
        tick += eps[-1]["num_steps"]
        k += 1
    assert k == meta["num_episodes"]
    g, st, extra = ograd.compute_grad(p, eps, args)
    for key in ("action_loss", "value_loss", "entropy"):
        assert np.isclose(st[key], meta[key], rtol=1e-9, atol=1e-9), key
    assert np.allclose(extra["returns"], z["returns"], rtol=1e-12, atol=1e-12)
    for key in z.files:
        if key.startswith("g_"):
            assert np.allclose(g[key[2:]], z[key], rtol=1e-8, atol=1e-10), key
        elif key.startswith("gsample_"):
            q = g[key[8:]]
            assert np.allclose(q.ravel()[::max(1, q.size // 2048)][:2048], z[key], rtol=1e-8, atol=1e-10), key


def test_tj_cfg_layout(built_lib):
    """vocab_type and its padding word sit at the end of ic3_tj_cfg (gcc probe against the ctypes mirror)."""
    from ic3net_b200 import _lib
    prog = ('#include <stdio.h>\n#include <stddef.h>\n#include "ic3net_b200.h"\nint main(){printf("%zu %zu %zu %d %d\\n",'
            'sizeof(ic3_tj_cfg), offsetof(ic3_tj_cfg, vocab_type), offsetof(ic3_tj_cfg, route_cells),'
            'IC3_TJ_VOCAB_BOOL, IC3_TJ_VOCAB_SCALAR);return 0;}')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "p.c"), "w").write(prog)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "p.c"), "-o",
                               os.path.join(d, "p")])
        size, off, off_cells, vb, vs = map(int, subprocess.check_output([os.path.join(d, "p")]).split())
    assert size == C.sizeof(_lib.TJCfg) and off == _lib.TJCfg.vocab_type.offset == off_cells + 8
    assert (vb, vs) == (_lib.TJ_VOCAB["bool"], _lib.TJ_VOCAB["scalar"])
    assert _lib.TJCfg().vocab_type == 0                       # zero-initialised structs keep the bool vocabulary


def scalar_cfg(**kw):
    from ic3net_b200 import _lib
    fake = 0x1000                                             # never dereferenced: validation fails first
    d = dict(B=4, N=5, vision=1, h=14, w=14, G=4, P=3, Lmax=20, outside_cls=0, car_cls=2, vocab=2, npath=12,
             env_id0=0, seed=1, grid=fake, route_len=fake, route_cells=fake, vocab_type=1)
    d.update(kw)
    return _lib.TJCfg(**d)


def fake_state():
    from ic3net_b200 import _lib
    f = 0x1000
    return _lib.TJState(loc=f, alive=f, wait=f, route_id=f, route_pos=f, last_act=f, completed=f, cars_in_sys=f,
                        has_failed=f, tick=f)


@pytest.mark.parametrize("kw", [dict(outside_cls=1), dict(car_cls=3), dict(vocab=3), dict(vocab_type=2),
                                dict(vocab_type=-1), dict(h=1), dict(w=1), dict(outside_cls=27, car_cls=29, vocab=30)])
def test_env_entry_points_refuse_bad_vocabularies(built_lib, kw):
    from ic3net_b200 import _lib
    lib = _lib.load()
    cfg, st = scalar_cfg(**kw), fake_state()
    assert lib.ic3_tj_obs(C.byref(cfg), C.byref(st), 0x1000, None) == E_RANGE
    assert lib.ic3_tj_obs_bounded(C.byref(cfg), C.byref(st), 0x1000, None) == E_RANGE
    assert lib.ic3_tj_reset(C.byref(cfg), C.byref(st), None, 0x1000, None) == E_RANGE
    assert lib.ic3_tj_step(C.byref(cfg), C.byref(st), 0x1000, 1, None, 0x1000, 0x1000, 0x1000, None, None) == E_RANGE


def policy_cfg(O, **kw):
    from ic3net_b200 import _lib
    hd = (C.c_int32 * _lib.MAX_HEADS)(2, 2, 0, 0)
    d = dict(B=4, N=5, H=128, O=O, nheads=2, head_dim=hd, hard_attn=1, comm_avg=1, comm_mask_zero=0, env_id0=0, seed=1,
             obs_off=0, obs_vocab=0, obs_ncount=0, cell=_lib.CELL_LSTM, passes=1, x_tanh=0, h_from_x=0)
    d.update(kw)
    return _lib.PolicyCfg(**d)


def test_encoder_entry_points_take_the_scalar_row_length(built_lib):
    from ic3net_b200 import _lib
    lib = _lib.load()
    f = 0x1000
    w = _lib.PolicyPacked(enc_wT=f, enc_b=f, c_wT=f, c_b=f, lstm_wT=f, lstm_b=f, head_w=f, head_b=f)
    env, st = scalar_cfg(), fake_state()
    O = 4 + 9 * 2
    for bad in (dict(O=2 + 9 * 2), dict(O=O, obs_off=4, obs_vocab=2, obs_ncount=1),       # a layout hint: refused
                dict(O=O, obs_off=2, obs_vocab=4, obs_ncount=1)):
        cfg = policy_cfg(**bad)
        assert lib.ic3_tj_encoder_index(C.byref(env), C.byref(st), C.byref(cfg), C.byref(w), f, None) == E_RANGE, bad
        assert lib.ic3_tj_obs_encode(C.byref(env), C.byref(st), C.byref(cfg), C.byref(w), f, f, None) == E_RANGE, bad
    bad_env = scalar_cfg(car_cls=1)
    cfg = policy_cfg(O)
    assert lib.ic3_tj_encoder_index(C.byref(bad_env), C.byref(st), C.byref(cfg), C.byref(w), f, None) == E_RANGE
    # no per-position table for the scalar vocabulary: it takes no layout hint
    assert lib.ic3_tj_encoder_table(C.byref(env), C.byref(cfg), C.byref(w), f, None) == E_RANGE
    # the tensor-core step's fused index encoder declines the scalar vocabulary
    io = _lib.PolicyIO(h=f, c=f, h_out=f, c_out=f, value=f, logp=f, workspace=f, err=f, comm_action=f,
                       **_lib.env_source(env, st))
    w.lstm_img, w.bias_cat, w.flags = f, f, f
    assert lib.ic3_policy_step(C.byref(cfg), C.byref(w), C.byref(io), None) == E_UNSUPPORTED


def test_gradient_kernels_do_not_cover_the_scalar_vocabulary(built_lib):
    """ic3_bptt_workspace_bytes and ic3_ff_grad_workspace_bytes are 0 for a scalar-vocabulary plan, with or without a
    layout hint, so grad_impl 'auto' takes autograd and 'kernels' / 'kernels_ff' refuse it."""
    from ic3net_b200 import _lib
    lib = _lib.load()
    env = scalar_cfg(vision=0, B=8, N=10, h=18, w=18)
    O = 4 + 2
    hints = (dict(), dict(obs_off=2, obs_vocab=4, obs_ncount=1), dict(obs_off=4, obs_vocab=4, obs_ncount=1))
    for hint in hints:
        for var in (dict(), dict(cell=_lib.CELL_TANH, comm_mask_zero=1, hard_attn=0)):
            cfg = policy_cfg(O, B=8, N=10, **dict(hint, **var))
            plan = _lib.BpttPlan(cfg=C.pointer(cfg), w=None, pp_env=None, tj_env=C.pointer(env), x_table=None,
                                 value_coeff=0.01, entr=0.0, workspace=None)
            assert lib.ic3_bptt_workspace_bytes(C.byref(plan)) == 0, (hint, var)
        cfg = policy_cfg(O, B=8, N=10, cell=_lib.CELL_TANH, x_tanh=1, h_from_x=1, passes=2, **hint)
        plan = _lib.FfGradPlan(cfg=C.pointer(cfg), w=None, pp_env=None, tj_env=C.pointer(env), value_coeff=0.01,
                               entr=0.0, max_rows=80, workspace=None)
        assert lib.ic3_ff_grad_workspace_bytes(C.byref(plan)) == 0, hint
    # the same plans on the bool vocabulary are covered: the scalar vocabulary is what excludes them
    V = 18 * 18 + 3
    benv = scalar_cfg(vision=0, B=8, N=10, h=18, w=18, outside_cls=V - 3, car_cls=V - 1, vocab=V, vocab_type=0)
    cfg = policy_cfg(2 + V, B=8, N=10, obs_off=2, obs_vocab=V, obs_ncount=1, cell=_lib.CELL_TANH, comm_mask_zero=1,
                     hard_attn=0)
    plan = _lib.BpttPlan(cfg=C.pointer(cfg), w=None, pp_env=None, tj_env=C.pointer(benv), x_table=None,
                         value_coeff=0.01, entr=0.0, workspace=None)
    assert lib.ic3_bptt_workspace_bytes(C.byref(plan)) > 0


def test_cli_accepts_the_scalar_vocabulary():
    from ic3net_b200 import main
    from ic3net_b200.utils import init_args_for_env
    argv = ["--env_name", "traffic_junction", "--vocab_type", "scalar"]
    parser = main.build_parser()
    init_args_for_env(parser, ["x"] + argv)                    # as main.main() adds the env's flags
    assert parser.parse_args(argv).vocab_type == "scalar"
