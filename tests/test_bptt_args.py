"""CPU tests of the agent-count checks at the BPTT entry points (ic3_bptt_workspace_bytes, ic3_bptt_begin,
ic3_bptt_prepare, ic3_bptt_step, ic3_bptt_finish, ic3_policy_step_backward): a plan whose agent count is out of range or
is not the environment's, whose observation width is not the environment's, or with no action head gets no workspace
and IC3_E_RANGE before any device work.  Every pointer but the plan's own structs is fake (never dereferenced), so a
call that got past the checks would launch kernels on them: nothing here may pass validation except the workspace
sizing of the valid plans."""
import ctypes as C

import pytest

FAKE = 0x1000
E_NULL, E_RANGE = -1, -2
TJ_H = TJ_W = 8
TJ_VOCAB = TJ_H * TJ_W + 3


def _setup(env="pp", cfg=None, pp=None, tj=None):
    """(lib, keep, calls): the six entry points bound to a plan on predator-prey (dim 3, vision 1) or traffic junction
    (8 x 8, vision 1) with 4 slots of 3 agents, the overrides applied to the policy config and the env config."""
    from ic3net_b200 import _lib
    lib = _lib.load()
    hd = (C.c_int32 * _lib.MAX_HEADS)(5, 2, 0, 0)
    pol = dict(B=4, N=3, H=128, nheads=2, head_dim=hd, hard_attn=1, comm_avg=1, comm_mask_zero=0, env_id0=0, seed=1,
               cell=_lib.CELL_LSTM, passes=1, x_tanh=0, h_from_x=0)
    if env == "pp":
        pol.update(O=9 * (3 * 3 + 4), obs_off=0, obs_vocab=3 * 3 + 4, obs_ncount=2)
        ecfg = _lib.PPCfg(**dict(dict(B=4, N=3, dim=3, vision=1, mode=0, naction=5, env_id0=0, enemy_comm=0, seed=1),
                                 **(pp or {})))
        pp_env, tj_env = C.pointer(ecfg), None
    else:
        pol.update(O=2 + 9 * TJ_VOCAB, obs_off=2, obs_vocab=TJ_VOCAB, obs_ncount=1)
        ecfg = _lib.TJCfg(**dict(dict(B=4, N=3, vision=1, h=TJ_H, w=TJ_W, G=4, P=3, Lmax=16, outside_cls=TJ_VOCAB - 3,
                                      car_cls=TJ_VOCAB - 1, vocab=TJ_VOCAB, npath=12, env_id0=0, seed=1, grid=FAKE,
                                      route_len=FAKE, route_cells=FAKE), **(tj or {})))
        pp_env, tj_env = None, C.pointer(ecfg)
    pol.update(cfg or {})
    pcfg = _lib.PolicyCfg(**pol)
    w = _lib.PolicyPacked(**{f: FAKE for f, _ in _lib.PolicyPacked._fields_})
    plan = _lib.BpttPlan(cfg=C.pointer(pcfg), w=C.pointer(w), pp_env=pp_env, tj_env=tj_env, x_table=FAKE,
                         value_coeff=0.01, entr=0.0, workspace=FAKE)
    pst = _lib.PPState(**{f: FAKE for f, _ in _lib.PPState._fields_})
    tst = _lib.TJState(**{f: FAKE for f, _ in _lib.TJState._fields_})
    state = dict(pp_state=C.pointer(pst)) if env == "pp" else dict(tj_state=C.pointer(tst))
    step = _lib.BpttStepIO(t=1, **dict({f: FAKE for f, t in _lib.BpttStepIO._fields_ if t is C.c_void_p}, **state))
    bwd = _lib.PolicyBwdIO(**dict({f: FAKE for f, t in _lib.PolicyBwdIO._fields_ if t is C.c_void_p}, **state))
    arr = lambda n: (C.c_void_p * n)(*[FAKE] * n)
    mk = lambda: _lib.PolicyParams(**dict({f: FAKE for f, t in _lib.PolicyParams._fields_ if t is C.c_void_p},
                                          head_w=arr(_lib.MAX_HEADS), head_b=arr(_lib.MAX_HEADS),
                                          c_w_pass=arr(_lib.MAX_PASSES), c_b_pass=arr(_lib.MAX_PASSES),
                                          f_w_pass=arr(_lib.MAX_PASSES), f_b_pass=arr(_lib.MAX_PASSES)))
    prm, grd = mk(), mk()
    keep = (ecfg, pcfg, w, plan, pst, tst, step, bwd, prm, grd)
    p = C.byref(plan)
    calls = {
        "ic3_bptt_begin": lambda: lib.ic3_bptt_begin(p, 1.0, None),
        "ic3_bptt_prepare": lambda: lib.ic3_bptt_prepare(p, C.byref(step), None),
        "ic3_bptt_step": lambda: lib.ic3_bptt_step(p, C.byref(step), None),
        "ic3_bptt_finish": lambda: lib.ic3_bptt_finish(p, C.byref(prm), C.byref(grd), FAKE, None),
        "ic3_policy_step_backward": lambda: lib.ic3_policy_step_backward(p, C.byref(bwd), C.byref(prm), C.byref(grd),
                                                                         None),
    }
    return lib, plan, keep, calls


ENTRY_POINTS = ["ic3_bptt_begin", "ic3_bptt_prepare", "ic3_bptt_step", "ic3_bptt_finish", "ic3_policy_step_backward"]

# (env kind, policy config overrides, env config overrides)
BAD = {
    "pp-N0": ("pp", dict(N=0), dict(N=0)),
    "tj-N0": ("tj", dict(N=0), dict(N=0)),
    "pp-N33": ("pp", dict(N=33), dict(N=33)),
    "tj-N33": ("tj", dict(N=33), dict(N=33)),
    "pp-N-not-env": ("pp", dict(N=4), {}),
    "tj-N-not-env": ("tj", dict(N=4), {}),
    "tj-N-below-env": ("tj", dict(N=2), {}),
    "pp-enemy-comm-without-prey-row": ("pp", {}, dict(enemy_comm=1)),
    "pp-32-predators": ("pp", dict(N=32), dict(N=32)),
    "pp-nheads0": ("pp", dict(nheads=0), {}),
    "tj-nheads0": ("tj", dict(nheads=0), {}),
    "pp-nheads5": ("pp", dict(nheads=5), {}),
    "pp-B0": ("pp", dict(B=0), dict(B=0)),
    "pp-O-not-env": ("pp", dict(O=9 * 13 + 1), {}),
    "tj-O-not-env": ("tj", dict(O=2 + 9 * TJ_VOCAB - 1), {}),
}


@pytest.mark.parametrize("env,cfg,ecfg", [("pp", {}, {}), ("tj", {}, {}), ("pp", dict(N=4), dict(N=3, enemy_comm=1)),
                                          ("tj", dict(N=32), dict(N=32)), ("pp", dict(N=1), dict(N=1)),
                                          ("tj", dict(N=1), dict(N=1)),
                                          ("pp", dict(N=32), dict(N=31, enemy_comm=1))])
def test_valid_plans_get_a_workspace(env, cfg, ecfg):
    """1 .. 32 agent rows, --enemy_comm's prey row included; sizing touches no device memory."""
    lib, plan, keep, _ = _setup(env, cfg, *((ecfg, None) if env == "pp" else (None, ecfg)))
    assert int(lib.ic3_bptt_workspace_bytes(C.byref(plan))) > 0


@pytest.mark.parametrize("case", sorted(BAD))
def test_bad_geometry_is_refused_before_device_work(case):
    env, cfg, ecfg = BAD[case]
    lib, plan, keep, calls = _setup(env, cfg, *((ecfg, None) if env == "pp" else (None, ecfg)))
    assert int(lib.ic3_bptt_workspace_bytes(C.byref(plan))) == 0, case
    for name in ENTRY_POINTS:
        assert calls[name]() == E_RANGE, (case, name)


def test_exactly_one_environment():
    lib, plan, keep, calls = _setup("pp")
    _, tplan, tkeep, _ = _setup("tj")
    plan.tj_env = tplan.tj_env                       # both set
    assert int(lib.ic3_bptt_workspace_bytes(C.byref(plan))) == 0
    for name in ENTRY_POINTS:
        assert calls[name]() == E_NULL, name
    plan.tj_env = None
    plan.pp_env = None                               # neither
    assert int(lib.ic3_bptt_workspace_bytes(C.byref(plan))) == 0
    for name in ENTRY_POINTS:
        assert calls[name]() == E_NULL, name
