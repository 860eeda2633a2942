"""CPU tests of the non-recurrent gradient entry points (ic3_ff_grad_*): the plan's layout, zero workspaces for the
configurations the kernels do not implement and IC3_E_* codes from the host-side checks, with no device work."""
import ctypes as C
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E_NULL, E_RANGE, E_UNSUPPORTED = -1, -2, -3


def setup():
    from ic3net_b200 import _lib
    lib = _lib.load()
    hd = (C.c_int32 * _lib.MAX_HEADS)(5, 0, 0, 0)
    D, v = 20, 1
    W = 2 * v + 1
    pol = dict(B=8, N=10, H=128, O=W * W * (D * D + 4), nheads=1, head_dim=hd, hard_attn=1, comm_avg=1,
               comm_mask_zero=0, env_id0=0, seed=1, obs_off=0, obs_vocab=D * D + 4, obs_ncount=2,
               cell=_lib.CELL_TANH, passes=2, x_tanh=1, h_from_x=1)
    env = dict(B=8, N=10, dim=D, vision=v, mode=0, naction=5, env_id0=0, enemy_comm=0, seed=1)
    return _lib, lib, pol, env


def nbytes(_lib, lib, pol, env, rows=80, **kw):
    cfg = _lib.PolicyCfg(**dict(pol, **kw))
    pp = _lib.PPCfg(**env)
    plan = _lib.FfGradPlan(cfg=C.pointer(cfg), w=None, pp_env=C.pointer(pp), tj_env=None, value_coeff=0.01, entr=0.0,
                           max_rows=rows, workspace=None)
    return int(lib.ic3_ff_grad_workspace_bytes(C.byref(plan))), plan, (cfg, pp)


def test_plan_layout_matches_header(tmp_path):
    from ic3net_b200 import _lib
    prog = ('#include <stdio.h>\n#include <stddef.h>\n#include "ic3net_b200.h"\n'
            'int main(){printf("%zu %zu %zu\\n", sizeof(ic3_ff_grad_plan), offsetof(ic3_ff_grad_plan, reserved0),'
            ' offsetof(ic3_ff_grad_plan, workspace)); return 0;}')
    c = tmp_path / "p.c"
    c.write_text(prog)
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(tmp_path / "p")])
    size, off, off_ws = map(int, subprocess.check_output([str(tmp_path / "p")]).split())
    assert size == C.sizeof(_lib.FfGradPlan)
    assert off == _lib.FfGradPlan.reserved0.offset and off_ws == _lib.FfGradPlan.workspace.offset
    assert off == _lib.FfGradPlan.max_rows.offset + 4 and off_ws == off + 4


def test_supported_configurations_get_a_workspace():
    _lib, lib, pol, env = setup()
    for kw in (dict(), dict(passes=1), dict(passes=4), dict(hard_attn=0, comm_avg=0), dict(comm_mask_zero=1, passes=1),
               dict(comm_mask_zero=1, passes=3)):
        assert nbytes(_lib, lib, pol, env, **kw)[0] > 0, kw
    small, _, _ = nbytes(_lib, lib, pol, env, rows=80)
    big, _, _ = nbytes(_lib, lib, pol, env, rows=800)
    assert big > small


@pytest.mark.parametrize("kw", [dict(H=64), dict(cell=0), dict(x_tanh=0), dict(h_from_x=0), dict(passes=5),
                                dict(nheads=2, head_dim=(C.c_int32 * 4)(5, 3, 0, 0)), dict(O=17)])
def test_out_of_scope_configurations_get_zero_bytes(kw):
    _lib, lib, pol, env = setup()
    assert nbytes(_lib, lib, pol, env, **kw)[0] == 0


def test_geometry_limits():
    _lib, lib, pol, env = setup()
    # a 7 x 7 window
    v = 3
    O = (2 * v + 1) ** 2 * (20 * 20 + 4)
    assert nbytes(_lib, lib, dict(pol, O=O), dict(env, vision=v))[0] == 0
    # an observation pattern wider than 512 columns: dim 23 -> 529 positions
    D = 23
    assert nbytes(_lib, lib, dict(pol, O=9 * (D * D + 4)), dict(env, dim=D))[0] == 0
    # 32 predators: beyond the index encoder (ic3_pp_encoder_index takes fewer than IC3_MAX_AGENTS)
    assert nbytes(_lib, lib, dict(pol, N=32), dict(env, N=32), rows=32 * 8)[0] == 0
    # a layout hint that is not the environment's
    assert nbytes(_lib, lib, dict(pol, obs_ncount=1), env)[0] == 0
    # capacity below one lock-step
    assert nbytes(_lib, lib, pol, env, rows=79)[0] == 0
    assert lib.ic3_ff_grad_workspace_bytes(None) == 0


def test_entry_points_check_arguments_before_device_work():
    _lib, lib, pol, env = setup()
    n, plan, keep = nbytes(_lib, lib, pol, env)
    assert n > 0
    assert lib.ic3_ff_grad_begin(None, None) == E_NULL
    assert lib.ic3_ff_grad_begin(C.byref(plan), None) == E_NULL              # no weights / workspace
    io = _lib.FfGradIO(nsteps=1)
    plan.workspace = 0x1000                                                  # never dereferenced
    w = _lib.PolicyPacked(f_wT=0x1000, c_wT=0x1000, head_w=0x1000)
    plan.w = C.pointer(w)
    assert lib.ic3_ff_grad_chunk(C.byref(plan), None, None) == E_NULL
    assert lib.ic3_ff_grad_chunk(C.byref(plan), C.byref(io), None) == E_NULL  # no records
    st = _lib.PPState(loc=0x1000)
    fake = dict(fresh=0x1000, logp=0x1000, action=0x1000, value=0x1000, ret=0x1000, adv=0x1000, alive_post=0x1000,
                pp_state=C.pointer(st), comm=0x1000)
    assert lib.ic3_ff_grad_chunk(C.byref(plan), C.byref(_lib.FfGradIO(nsteps=2, **fake)), None) == E_RANGE  # > capacity
    assert lib.ic3_ff_grad_chunk(C.byref(plan), C.byref(_lib.FfGradIO(nsteps=0, **fake)), None) == E_RANGE
    assert lib.ic3_ff_grad_finish(C.byref(plan), None, None, None, None) == E_NULL
    cfg, pp = keep
    cfg.x_tanh = 0
    assert lib.ic3_ff_grad_chunk(C.byref(plan), C.byref(_lib.FfGradIO(nsteps=1, **fake)), None) == E_UNSUPPORTED
    p = _lib.PolicyParams()
    assert lib.ic3_ff_grad_finish(C.byref(plan), C.byref(p), C.byref(p), 0x1000, None) == E_UNSUPPORTED


def test_cli_accepts_kernels_ff():
    from ic3net_b200 import main
    assert main.build_parser().parse_args(["--grad_impl", "kernels_ff"]).grad_impl == "kernels_ff"
