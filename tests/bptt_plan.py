"""A BPTT plan with fake device pointers (never dereferenced) for the CPU tests of the entry points' argument checks.
Not a test module: tests/test_bptt_args.py and tests/test_graph_update_abi.py build their plans here."""
import ctypes as C

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
