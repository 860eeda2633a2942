"""CPU tests of the agent-count checks at the BPTT entry points (ic3_bptt_workspace_bytes, ic3_bptt_begin,
ic3_bptt_prepare, ic3_bptt_step, ic3_bptt_finish, ic3_policy_step_backward): a plan whose agent count is out of range or
is not the environment's, whose observation width is not the environment's, or with no action head gets no workspace
and IC3_E_RANGE before any device work.  Every pointer but the plan's own structs is fake (never dereferenced), so a
call that got past the checks would launch kernels on them: nothing here may pass validation except the workspace
sizing of the valid plans."""
import ctypes as C

import pytest

from bptt_plan import E_NULL, E_RANGE, TJ_VOCAB, _setup

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
