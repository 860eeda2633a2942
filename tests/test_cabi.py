"""CPU tests of the boundary: the C-ABI library builds for sm_90a, loads, and exports
every symbol include/ic3net_b200.h declares (no compute calls without a GPU)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "ic3net_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ic3_[a-z0-9_]+)\s*\(", src)))


def test_header_and_binding_agree():
    from ic3net_b200 import _lib
    assert header_symbols() == sorted(_lib.SYMBOLS)


def test_library_exports_every_symbol(built_lib):
    lib = ctypes.CDLL(built_lib)
    for name in header_symbols():
        assert hasattr(lib, name), name
    lib.ic3_version.restype = ctypes.c_char_p
    assert b"sm_90a" in lib.ic3_version()
    lib.ic3_strerror.restype = ctypes.c_char_p
    assert b"NULL" in lib.ic3_strerror(-1)


def test_struct_sizes_match_header(built_lib):
    """ctypes mirrors must have the C layout (checked with a tiny gcc probe)."""
    import subprocess
    import tempfile
    from ic3net_b200 import _lib
    names = {"ic3_pp_cfg": _lib.PPCfg, "ic3_pp_state": _lib.PPState, "ic3_rollout_io": _lib.RolloutIO,
             "ic3_tj_cfg": _lib.TJCfg, "ic3_tj_state": _lib.TJState, "ic3_policy_cfg": _lib.PolicyCfg,
             "ic3_policy_params": _lib.PolicyParams, "ic3_policy_packed": _lib.PolicyPacked,
             "ic3_policy_io": _lib.PolicyIO, "ic3_bptt_plan": _lib.BpttPlan, "ic3_bptt_step_io": _lib.BpttStepIO,
             "ic3_ff_grad_plan": _lib.FfGradPlan, "ic3_ff_grad_io": _lib.FfGradIO}
    prog = '#include <stdio.h>\n#include "ic3net_b200.h"\nint main(){' + "".join(
        'printf("%s %%zu\\n", sizeof(%s));' % (n, n) for n in names) + "return 0;}"
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(prog)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", os.path.join(d, "p")])
        out = subprocess.check_output([os.path.join(d, "p")]).decode().split("\n")
    sizes = dict(l.split() for l in out if l)
    for n, cls in names.items():
        assert int(sizes[n]) == ctypes.sizeof(cls), n


def test_no_cpu_fallback():
    """Product modules must refuse to run without CUDA instead of falling back."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import argparse
    from ic3net_b200.predator_prey_env import PredatorPreyEnv
    a = argparse.Namespace(dim=5, vision=0, moving_prey=False, mode="mixed", enemy_comm=False, nenemies=1,
                           nfriendly=3, nagents=3, no_stay=False, nenvs=2, seed=0)
    with pytest.raises(RuntimeError):
        PredatorPreyEnv().multi_agent_init(a)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "ic3net_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", txt, flags=re.M), f


def test_entry_points_validate_arguments_before_touching_the_device(built_lib):
    """Error behaviour of the boundary: a bad call returns IC3_E_NULL / IC3_E_RANGE / IC3_E_UNSUPPORTED from the host-side
    checks (the conditions under which the reference raises -- wrong mode predator_prey_env.py:269, too many agents -- or
    configurations the kernels do not implement); nothing is launched, so this runs without a GPU."""
    from ic3net_b200 import _lib
    lib = _lib.load()
    E_NULL, E_RANGE, E_UNSUPPORTED = -1, -2, -3
    fake = 0x1000                      # never dereferenced: validation fails first
    st = _lib.PPState(loc=fake, reached=fake, done=fake, success=fake, episode=fake, tick=fake)
    ok = dict(B=4, N=3, dim=5, vision=1, mode=0, naction=5, env_id0=0, enemy_comm=0, seed=1)
    assert lib.ic3_pp_step(None, ctypes.byref(st), fake, 1, fake, None, fake, None, None) == E_NULL
    assert lib.ic3_pp_reset(ctypes.byref(_lib.PPCfg(**ok)), ctypes.byref(_lib.PPState()), None, None, None) == E_NULL
    for bad in (dict(N=32), dict(N=0), dict(mode=3), dict(naction=6), dict(dim=200), dict(vision=8), dict(dim=1)):
        cfg = _lib.PPCfg(**dict(ok, **bad))
        assert lib.ic3_pp_step(ctypes.byref(cfg), ctypes.byref(st), fake, 1, fake, None, fake, None, None) == E_RANGE, bad
    assert lib.ic3_pp_step(ctypes.byref(_lib.PPCfg(**ok)), ctypes.byref(st), None, 1, fake, None, fake, None,
                           None) == E_NULL                   # no actions
    # policy: hidden sizes / head layouts the kernels do not cover
    hd = (ctypes.c_int32 * _lib.MAX_HEADS)(5, 2, 0, 0)
    pol = dict(B=4, N=3, H=128, O=29, nheads=2, head_dim=hd, hard_attn=1, comm_avg=1, comm_mask_zero=0, env_id0=0, seed=1,
               obs_off=0, obs_vocab=0, obs_ncount=0, cell=_lib.CELL_LSTM, passes=1, x_tanh=0, h_from_x=0)
    w, io = _lib.PolicyPacked(), _lib.PolicyIO()
    call = lambda **kw: lib.ic3_policy_step(ctypes.byref(_lib.PolicyCfg(**dict(pol, **kw))), ctypes.byref(w),
                                            ctypes.byref(io), None)
    assert call(H=100) == E_UNSUPPORTED and call(nheads=0) == E_RANGE and call(N=33) == E_RANGE
    assert call(passes=_lib.MAX_PASSES + 1) == E_RANGE and call(cell=7) == E_RANGE
    assert call() == E_NULL                                   # valid configuration, but no packed weights / buffers
    assert lib.ic3_policy_step(None, ctypes.byref(w), ctypes.byref(io), None) == E_NULL
    assert lib.ic3_policy_workspace_bytes(ctypes.byref(_lib.PolicyCfg(**dict(pol, H=64)))) == 0    # SIMT: no workspace
    assert lib.ic3_policy_workspace_bytes(ctypes.byref(_lib.PolicyCfg(**pol))) > 0
    assert lib.ic3_bptt_workspace_bytes(None) == 0
    assert lib.ic3_sample_actions(ctypes.byref(_lib.PolicyCfg(**pol)), None, None, None, None, None) == E_NULL
    for code, word in ((E_RANGE, b"range"), (E_UNSUPPORTED, b"not implemented"), (0, b"ok")):
        assert word in lib.ic3_strerror(code)
    with pytest.raises(RuntimeError, match="range"):
        _lib.check(E_RANGE)
