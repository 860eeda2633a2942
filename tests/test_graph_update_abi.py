"""CPU tests of the entry points graph_update captures (ic3_bptt_begin_dev, ic3_rmsprop_step_dev): null pointers and
bad sizes are refused with IC3_E_* before any device work.  Every pointer is fake (never dereferenced), so a call that
got past the checks would launch kernels on them: nothing here may pass validation."""
import ctypes as C

import pytest

from bptt_plan import FAKE, _setup

E_NULL, E_RANGE = -1, -2


def test_declared_and_flag_bit():
    from ic3net_b200 import _lib
    assert {"ic3_bptt_begin_dev", "ic3_rmsprop_step_dev"} <= set(_lib.SYMBOLS)
    assert _lib.ERR_GRAD_DIV == 0x400


@pytest.mark.parametrize("case, want", [
    ("no_plan", E_NULL), ("no_c", E_NULL), ("empty_c", E_RANGE), ("negative_n", E_RANGE), ("bad_agents", E_RANGE),
    ("no_workspace", E_NULL)])
def test_bptt_begin_dev_refuses(case, want):
    lib, plan, keep, _ = _setup(cfg=dict(N=0) if case == "bad_agents" else None)
    if case == "no_workspace":
        plan.workspace = None
    c, n = FAKE, 1024
    if case == "no_c":
        c = None
    elif case == "empty_c":
        n = 0
    elif case == "negative_n":
        n = -4
    p = None if case == "no_plan" else C.byref(plan)
    assert lib.ic3_bptt_begin_dev(p, c, n, None) == want


@pytest.mark.parametrize("case, want", [
    ("no_stat", E_NULL), ("no_grad", E_NULL), ("no_param", E_NULL), ("no_square_avg", E_NULL), ("no_err", E_NULL),
    ("zero_n", E_RANGE), ("zero_eps", E_RANGE), ("misaligned", E_RANGE)])
def test_rmsprop_step_dev_refuses(case, want):
    from ic3net_b200 import _lib
    lib = _lib.load()
    a = dict(n=1024, lr=1e-3, alpha=0.97, eps=1e-6, stat=FAKE, grad=FAKE, param=FAKE, sq=FAKE, err=FAKE)
    if case.startswith("no_"):
        a[{"square_avg": "sq"}.get(case[3:], case[3:])] = None
    elif case == "zero_n":
        a["n"] = 0
    elif case == "zero_eps":
        a["eps"] = 0.0
    else:
        a["grad"] = FAKE + 4
    assert lib.ic3_rmsprop_step_dev(a["n"], a["lr"], a["alpha"], a["eps"], a["stat"], a["grad"], a["param"], a["sq"],
                                    a["err"], None) == want
