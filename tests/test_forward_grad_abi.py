"""CPU test of the C boundary of the differentiable forward (ic3_policy_step_backward): the ctypes mirror of
ic3_policy_bwd_io has the header's members, size and offsets, and bad arguments are refused with IC3_E_* before any
device work (nothing here launches a kernel, so it runs without a GPU)."""
import ctypes
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 0x1000                  # never dereferenced: validation fails first


def test_policy_bwd_io_layout_matches_header(tmp_path):
    from ic3net_b200 import _lib
    fields = [f for f, _ in _lib.PolicyBwdIO._fields_]
    src = open(os.path.join(ROOT, "include", "ic3net_b200.h")).read()
    body = re.search(r"typedef struct \{((?:(?!typedef struct).)*?)\} ic3_policy_bwd_io;", src, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert re.findall(r"\b(\w+);", body) == fields            # same members, same order
    assert re.search(r"int ic3_policy_step_backward\(const ic3_bptt_plan\* plan, const ic3_policy_bwd_io\* io,", src)
    prog = '#include <stdio.h>\n#include <stddef.h>\n#include "ic3net_b200.h"\nint main(){' + \
           'printf("%zu\\n", sizeof(ic3_policy_bwd_io));' + \
           "".join('printf("%%zu\\n", offsetof(ic3_policy_bwd_io, %s));' % f for f in fields) + 'return 0;}'
    c = tmp_path / "p.c"
    c.write_text(prog)
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(tmp_path / "p")])
    out = [int(v) for v in subprocess.check_output([str(tmp_path / "p")]).decode().split()]
    assert out[0] == ctypes.sizeof(_lib.PolicyBwdIO)
    assert out[1:] == [getattr(_lib.PolicyBwdIO, f).offset for f in fields]


def _setup(**over):
    """A plan, io, params and grads that pass every check (all pointers fake), then the overrides."""
    from ic3net_b200 import _lib
    hd = (ctypes.c_int32 * _lib.MAX_HEADS)(5, 2, 0, 0)
    pol = dict(B=4, N=3, H=128, O=4 * 13 * 9, nheads=2, head_dim=hd, hard_attn=1, comm_avg=1, comm_mask_zero=0,
               env_id0=0, seed=1, obs_off=0, obs_vocab=13, obs_ncount=2, cell=_lib.CELL_LSTM, passes=1, x_tanh=0,
               h_from_x=0)
    pol.update(over.pop("cfg", {}))
    cfg = _lib.PolicyCfg(**pol)
    env = _lib.PPCfg(B=4, N=3, dim=3, vision=1, mode=0, naction=5, env_id0=0, enemy_comm=0, seed=1)
    w = _lib.PolicyPacked(**{f: FAKE for f, _ in _lib.PolicyPacked._fields_})
    plan = _lib.BpttPlan(cfg=ctypes.pointer(cfg), w=ctypes.pointer(w), pp_env=ctypes.pointer(env), tj_env=None,
                         x_table=FAKE, value_coeff=0.0, entr=0.0, workspace=FAKE)
    st = _lib.PPState(loc=FAKE)
    io = _lib.PolicyBwdIO(h_prev=FAKE, c_prev=FAKE, h_new=FAKE, logp=FAKE, comm=FAKE, alive=None,
                          pp_state=ctypes.pointer(st), dh_prev=FAKE, dc_prev=FAKE)
    arr = lambda n: (ctypes.c_void_p * n)(*[FAKE] * n)
    mk = lambda: _lib.PolicyParams(**{f: FAKE for f in ("encoder_w", "encoder_b", "c_w", "c_b", "w_ih", "w_hh", "b_ih",
                                                        "b_hh", "value_w", "value_b")},
                                   head_w=arr(_lib.MAX_HEADS), head_b=arr(_lib.MAX_HEADS), c_w_pass=arr(_lib.MAX_PASSES),
                                   c_b_pass=arr(_lib.MAX_PASSES), f_w_pass=arr(_lib.MAX_PASSES),
                                   f_b_pass=arr(_lib.MAX_PASSES))
    keep = (cfg, env, w, st)
    return plan, io, mk(), mk(), keep


def test_bad_arguments_are_refused_before_device_work(built_lib):
    from ic3net_b200 import _lib
    lib = _lib.load()
    E_NULL, E_RANGE, E_UNSUPPORTED = -1, -2, -3

    def call(plan, io, params, grads):
        return lib.ic3_policy_step_backward(plan and ctypes.byref(plan), io and ctypes.byref(io),
                                            params and ctypes.byref(params), grads and ctypes.byref(grads), None)

    plan, io, prm, grd, keep = _setup()
    assert call(None, io, prm, grd) == E_NULL
    assert call(plan, None, prm, grd) == E_NULL
    assert call(plan, io, None, grd) == E_NULL
    assert call(plan, io, prm, None) == E_NULL
    for field in ("h_prev", "h_new", "logp", "dh_prev", "c_prev", "dc_prev", "comm"):
        plan, io, prm, grd, keep = _setup()
        setattr(io, field, None)
        assert call(plan, io, prm, grd) == E_NULL, field
    plan, io, prm, grd, keep = _setup()
    io.pp_state = None                               # the copied env state is required
    assert call(plan, io, prm, grd) == E_NULL
    plan, io, prm, grd, keep = _setup()
    plan.x_table = None                              # the LSTM cell's operands need the per-position encoder table
    assert call(plan, io, prm, grd) == E_NULL
    plan, io, prm, grd, keep = _setup()
    plan.workspace = None
    assert call(plan, io, prm, grd) == E_NULL
    plan, io, prm, grd, keep = _setup()
    grd.w_ih = None                                  # a gradient buffer ic3_bptt_finish would write
    assert call(plan, io, prm, grd) == E_NULL
    plan, io, prm, grd, keep = _setup()
    grd.head_w[1] = None
    assert call(plan, io, prm, grd) == E_NULL
    for cfg in (dict(H=64), dict(obs_vocab=0), dict(x_tanh=1), dict(h_from_x=1), dict(passes=_lib.MAX_PASSES + 1),
                dict(cell=_lib.CELL_TANH),          # the tanh cell without comm_mask_zero / with hard attention
                dict(nheads=3, head_dim=(ctypes.c_int32 * _lib.MAX_HEADS)(5, 2, 1, 0))):      # 8 action logits + value
        plan, io, prm, grd, keep = _setup(cfg=cfg)
        assert call(plan, io, prm, grd) in (E_RANGE, E_UNSUPPORTED), cfg
    # the tanh RNN (IC / IRIC) needs no c, no table and no LSTM gradient buffers -- but its f_w gradient
    tanh = dict(cell=_lib.CELL_TANH, comm_mask_zero=1, hard_attn=0)
    plan, io, prm, grd, keep = _setup(cfg=tanh)
    grd.f_w_pass[0] = None
    assert call(plan, io, prm, grd) == E_NULL
    plan, io, prm, grd, keep = _setup(cfg=tanh)
    plan.w.contents.f_wT = None
    assert call(plan, io, prm, grd) == E_NULL
