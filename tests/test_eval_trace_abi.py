"""CPU tests of the evaluation recorder's entry points (ic3_trace_step / ic3_comm_map_step): a bad call is refused by
the host-side checks with the ABI's error codes before anything is launched, and Trainer.evaluate_trace's slot lists are
checked in Python."""
import ctypes

import pytest

E_NULL, E_RANGE, E_ARG = -1, -2, -4
FAKE = 0x1000                      # never dereferenced: validation fails first


def _io(_lib, tj=False):
    if tj:
        env = _lib.TJCfg(B=4, N=3, vision=1, h=14, w=14, G=4, P=3, Lmax=20, outside_cls=11, car_cls=13, vocab=14,
                         npath=12, env_id0=0, seed=1, grid=FAKE, route_len=FAKE, route_cells=FAKE)
        st = _lib.TJState(loc=FAKE, alive=FAKE, wait=FAKE, route_id=FAKE, route_pos=FAKE, last_act=FAKE,
                          completed=FAKE, cars_in_sys=FAKE, has_failed=FAKE, tick=FAKE)
        src = dict(tj_env=ctypes.pointer(env), tj_state=ctypes.pointer(st))
    else:
        env = _lib.PPCfg(B=4, N=3, dim=5, vision=1, mode=0, naction=5, env_id0=0, enemy_comm=0, seed=1)
        st = _lib.PPState(loc=FAKE, reached=FAKE, done=FAKE, success=FAKE, episode=FAKE, tick=FAKE)
        src = dict(pp_env=ctypes.pointer(env), pp_state=ctypes.pointer(st))
    io = _lib.EvalStepIO(nheads=2, logp_cols=7, comm_col=6, max_steps=20, t_ep=FAKE, halted=FAKE, action=FAKE,
                         value=FAKE, logp=FAKE, reward=FAKE, fresh=FAKE, out_loc=FAKE, out_success=FAKE, err=FAKE, **src)
    tr = _lib.EvalTrace(T=40, K=2, slots=FAKE, loc=FAKE, loc_next=FAKE, alive=FAKE, action=FAKE, value=FAKE,
                        reward=FAKE, t_ep=FAKE, done=FAKE, success=FAKE, valid=FAKE, comm_prob=FAKE,
                        route_id=FAKE if tj else None)
    return io, tr, (env, st)


def _copy(cls, s, **over):
    c = cls.from_buffer_copy(s)
    for k, v in over.items():
        setattr(c, k, v)
    return c


@pytest.mark.parametrize("tj", [False, True], ids=["pp", "tj"])
def test_trace_step_checks_arguments(built_lib, tj):
    from ic3net_b200 import _lib
    lib = _lib.load()
    io, tr, keep = _io(_lib, tj)
    call = lambda i=io, r=tr, t=0: lib.ic3_trace_step(ctypes.byref(i), ctypes.byref(r), t, None)
    assert lib.ic3_trace_step(None, ctypes.byref(tr), 0, None) == E_NULL
    assert lib.ic3_trace_step(ctypes.byref(io), None, 0, None) == E_NULL
    for field in ("t_ep", "halted", "action", "value", "reward", "fresh", "out_loc", "out_success", "err", "logp"):
        assert call(i=_copy(_lib.EvalStepIO, io, **{field: None})) == E_NULL, field
    for field in ("slots", "loc", "loc_next", "alive", "action", "value", "reward", "t_ep", "done", "success", "valid",
                  "comm_prob"):
        assert call(r=_copy(_lib.EvalTrace, tr, **{field: None})) == E_NULL, field
    # neither or both environments
    assert call(i=_copy(_lib.EvalStepIO, io, pp_env=None, tj_env=None)) == E_NULL
    both = _copy(_lib.EvalStepIO, io)
    other = _io(_lib, not tj)[0]
    both.pp_env, both.pp_state, both.tj_env, both.tj_state = (io.pp_env or other.pp_env, io.pp_state or other.pp_state,
                                                              io.tj_env or other.tj_env, io.tj_state or other.tj_state)
    assert call(i=both) == E_NULL
    for field, bad in (("nheads", 0), ("nheads", 5), ("max_steps", 0), ("max_steps", 32768), ("comm_col", 7),
                       ("comm_col", -2)):
        assert call(i=_copy(_lib.EvalStepIO, io, **{field: bad})) == E_RANGE, (field, bad)
    for field, bad in (("T", 0), ("K", 0)):
        assert call(r=_copy(_lib.EvalTrace, tr, **{field: bad})) == E_RANGE, field
    assert call(t=-1) == E_RANGE and call(t=41) == E_RANGE
    # a gate probability without a gate, a route record on predator-prey / none on traffic junction
    assert call(i=_copy(_lib.EvalStepIO, io, comm_col=-1)) == E_ARG
    assert call(r=_copy(_lib.EvalTrace, tr, route_id=None if tj else FAKE)) == (E_NULL if tj else E_ARG)


@pytest.mark.parametrize("tj", [False, True], ids=["pp", "tj"])
def test_comm_map_step_checks_arguments(built_lib, tj):
    from ic3net_b200 import _lib
    lib = _lib.load()
    io, _, keep = _io(_lib, tj)
    call = lambda i=io, c=FAKE: lib.ic3_comm_map_step(ctypes.byref(i), c, None)
    assert call(c=None) == E_NULL
    assert lib.ic3_comm_map_step(None, FAKE, None) == E_NULL
    for field in ("t_ep", "halted", "action"):
        assert call(i=_copy(_lib.EvalStepIO, io, **{field: None})) == E_NULL, field
    for field, bad in (("nheads", 0), ("max_steps", 0), ("comm_col", 9)):
        assert call(i=_copy(_lib.EvalStepIO, io, **{field: bad})) == E_RANGE, field
    cfg = io.tj_env.contents if tj else io.pp_env.contents
    saved = cfg.B
    cfg.B = 0
    assert call() == E_RANGE
    cfg.B = saved


def test_slot_lists_are_checked_in_python():
    from ic3net_b200.eval_trace import parse_slots
    assert parse_slots(3, 10) == (0, 1, 2) and parse_slots([9, 0, 4], 10) == (9, 0, 4)
    for bad in (0, 11, [], [1, 1], [10], [-1]):
        with pytest.raises(ValueError):
            parse_slots(bad, 10)
