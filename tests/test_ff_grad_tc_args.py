"""CPU tests of the tensor-core form of the non-recurrent gradient (ic3_ff_grad_plan.impl = IC3_FF_GRAD_TC): the plan's
layout, and a workspace for exactly the configurations the SIMT form (impl 0) covers."""
import ctypes as C
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


def nbytes(pol, env, impl, rows=80, **kw):
    from ic3net_b200 import _lib
    cfg = _lib.PolicyCfg(**dict(pol, **kw))
    pp = _lib.PPCfg(**env)
    plan = _lib.FfGradPlan(cfg=C.pointer(cfg), w=None, pp_env=C.pointer(pp), tj_env=None, value_coeff=0.01, entr=0.0,
                           max_rows=rows, impl=impl, workspace=None)
    return int(_lib.load().ic3_ff_grad_workspace_bytes(C.byref(plan)))


def test_plan_layout_matches_header(tmp_path):
    from ic3net_b200 import _lib
    prog = ('#include <stdio.h>\n#include <stddef.h>\n#include "ic3net_b200.h"\n'
            'int main(){printf("%zu %zu %zu %d %d\\n", sizeof(ic3_ff_grad_plan), offsetof(ic3_ff_grad_plan, impl),'
            ' offsetof(ic3_ff_grad_plan, workspace), (int)IC3_FF_GRAD_SIMT, (int)IC3_FF_GRAD_TC); return 0;}')
    c = tmp_path / "p.c"
    c.write_text(prog)
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(tmp_path / "p")])
    size, off, off_ws, simt, tc = map(int, subprocess.check_output([str(tmp_path / "p")]).split())
    assert size == C.sizeof(_lib.FfGradPlan)
    assert off == _lib.FfGradPlan.impl.offset and off_ws == _lib.FfGradPlan.workspace.offset
    # the field took the place of the former padding word: the struct keeps its size and offsets
    assert off == _lib.FfGradPlan.max_rows.offset + 4 and off_ws == off + 4
    assert (simt, tc) == (_lib.FF_GRAD_SIMT, _lib.FF_GRAD_TC) == (0, 1)
    assert _lib.FfGradPlan().impl == _lib.FF_GRAD_SIMT           # zero-initialised plans keep the SIMT kernels


def test_same_coverage_as_the_simt_kernels():
    """Every configuration test_ff_grad_args.py covers gets a workspace with impl 1 as well (more than impl 0's: the
    weight images), at every capacity."""
    _lib, lib, pol, env = setup()
    for kw in (dict(), dict(passes=1), dict(passes=4), dict(hard_attn=0, comm_avg=0), dict(comm_mask_zero=1, passes=1),
               dict(comm_mask_zero=1, passes=3)):
        simt, tc = nbytes(pol, env, 0, **kw), nbytes(pol, env, 1, **kw)
        assert simt > 0 and tc > simt, kw
    assert nbytes(pol, env, 1, rows=800) > nbytes(pol, env, 1, rows=80)


@pytest.mark.parametrize("kw", [dict(H=64), dict(cell=0), dict(x_tanh=0), dict(h_from_x=0), dict(passes=5),
                                dict(nheads=2, head_dim=(C.c_int32 * 4)(5, 3, 0, 0)), dict(O=17)])
def test_out_of_scope_configurations_get_zero_bytes(kw):
    _lib, lib, pol, env = setup()
    assert nbytes(pol, env, 0, **kw) == 0 and nbytes(pol, env, 1, **kw) == 0


def test_geometry_limits():
    _lib, lib, pol, env = setup()
    v = 3                                                     # a 7 x 7 window
    assert nbytes(dict(pol, O=(2 * v + 1) ** 2 * (20 * 20 + 4)), dict(env, vision=v), 1) == 0
    D = 23                                                    # 529 positions: a pattern wider than 512 columns
    assert nbytes(dict(pol, O=9 * (D * D + 4)), dict(env, dim=D), 1) == 0
    assert nbytes(dict(pol, N=32), dict(env, N=32), 1, rows=32 * 8) == 0
    assert nbytes(dict(pol, obs_ncount=1), env, 1) == 0         # a layout hint that is not the environment's
    assert nbytes(pol, env, 1, rows=79) == 0                    # capacity below one lock-step


@pytest.mark.parametrize("impl", [2, -1, 1 << 20])
def test_unknown_impl_gets_zero_bytes_and_no_device_work(impl):
    _lib, lib, pol, env = setup()
    assert nbytes(pol, env, impl) == 0
    cfg, pp = _lib.PolicyCfg(**pol), _lib.PPCfg(**env)
    w = _lib.PolicyPacked(f_wT=0x1000, c_wT=0x1000, head_w=0x1000)
    plan = _lib.FfGradPlan(cfg=C.pointer(cfg), w=C.pointer(w), pp_env=C.pointer(pp), tj_env=None, value_coeff=0.01,
                           entr=0.0, max_rows=80, impl=impl, workspace=0x1000)
    E_UNSUPPORTED = -3
    assert lib.ic3_ff_grad_begin(C.byref(plan), None) == E_UNSUPPORTED
    st = _lib.PPState(loc=0x1000)
    io = _lib.FfGradIO(nsteps=1, fresh=0x1000, logp=0x1000, action=0x1000, value=0x1000, ret=0x1000, adv=0x1000,
                       alive_post=0x1000, comm=0x1000, pp_state=C.pointer(st))
    assert lib.ic3_ff_grad_chunk(C.byref(plan), C.byref(io), None) == E_UNSUPPORTED
    p = _lib.PolicyParams()
    assert lib.ic3_ff_grad_finish(C.byref(plan), C.byref(p), C.byref(p), 0x1000, None) == E_UNSUPPORTED


def test_scalar_vocabulary_gets_zero_bytes():
    from ic3net_b200 import _lib
    lib = _lib.load()
    fake = 0x1000
    env = _lib.TJCfg(B=8, N=10, vision=0, h=18, w=18, G=4, P=3, Lmax=20, outside_cls=0, car_cls=2, vocab=2, npath=12,
                     env_id0=0, seed=1, grid=fake, route_len=fake, route_cells=fake, vocab_type=_lib.TJ_VOCAB["scalar"])
    hd = (C.c_int32 * _lib.MAX_HEADS)(2, 2, 0, 0)
    for hint in (dict(obs_off=0, obs_vocab=0, obs_ncount=0), dict(obs_off=2, obs_vocab=4, obs_ncount=1)):
        cfg = _lib.PolicyCfg(B=8, N=10, H=128, O=4 + 2, nheads=2, head_dim=hd, hard_attn=1, comm_avg=1, comm_mask_zero=0,
                             env_id0=0, seed=1, cell=_lib.CELL_TANH, passes=2, x_tanh=1, h_from_x=1, **hint)
        plan = _lib.FfGradPlan(cfg=C.pointer(cfg), w=None, pp_env=None, tj_env=C.pointer(env), value_coeff=0.01,
                               entr=0.0, max_rows=80, impl=_lib.FF_GRAD_TC, workspace=None)
        assert lib.ic3_ff_grad_workspace_bytes(C.byref(plan)) == 0, hint


def test_cli_accepts_kernels_ff_tc():
    from ic3net_b200 import main
    assert main.build_parser().parse_args(["--grad_impl", "kernels_ff_tc"]).grad_impl == "kernels_ff_tc"
