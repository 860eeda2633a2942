"""CPU tests of the message recorder's entry points (ic3_trace_comm_step / ic3_message_map_step): a bad call is refused
by the host-side checks with the ABI's error codes before anything is launched; and the host side of the message map
(its blocks, scale and means)."""
import ctypes

import numpy as np
import pytest

E_NULL, E_RANGE = -1, -2
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
    cm = _lib.EvalCommIO(h=FAKE, comm=FAKE, alive=FAKE, fresh=FAKE, H=128, comm_avg=1, hard=1)
    tr = _lib.EvalTrace(T=40, K=2, slots=FAKE)
    return io, cm, tr, (env, st)


def _copy(cls, s, **over):
    c = cls.from_buffer_copy(s)
    for k, v in over.items():
        setattr(c, k, v)
    return c


def _comm_refusals(_lib, call, io, cm):
    """The refusals both entry points share: the step io, the comm io's pointers and ranges."""
    for field in ("t_ep", "halted", "action"):
        assert call(i=_copy(_lib.EvalStepIO, io, **{field: None})) == E_NULL, field
    assert call(i=_copy(_lib.EvalStepIO, io, pp_env=None, tj_env=None)) == E_NULL
    for field in ("h", "alive", "fresh", "comm"):
        assert call(c=_copy(_lib.EvalCommIO, cm, **{field: None})) == E_NULL, field
    for field, bad in (("H", 0), ("H", 8), ("H", 24), ("H", 1040), ("comm_avg", 2), ("comm_avg", -1), ("hard", 2)):
        assert call(c=_copy(_lib.EvalCommIO, cm, **{field: bad})) == E_RANGE, (field, bad)
    for field, bad in (("nheads", 0), ("max_steps", 0), ("comm_col", 9)):
        assert call(i=_copy(_lib.EvalStepIO, io, **{field: bad})) == E_RANGE, (field, bad)
    cfg = io.tj_env.contents if io.tj_env else io.pp_env.contents
    saved = cfg.B
    cfg.B = 0
    assert call() == E_RANGE
    cfg.B = saved


@pytest.mark.parametrize("tj", [False, True], ids=["pp", "tj"])
def test_trace_comm_step_checks_arguments(built_lib, tj):
    from ic3net_b200 import _lib
    lib = _lib.load()
    io, cm, tr, keep = _io(_lib, tj)

    def call(i=io, c=cm, r=tr, h=FAKE, g=FAKE, s=FAKE, t=0):
        return lib.ic3_trace_comm_step(ctypes.byref(i), ctypes.byref(c), ctypes.byref(r), h, g, s, t, None)
    assert lib.ic3_trace_comm_step(None, ctypes.byref(cm), ctypes.byref(tr), FAKE, FAKE, FAKE, 0, None) == E_NULL
    assert lib.ic3_trace_comm_step(ctypes.byref(io), None, ctypes.byref(tr), FAKE, FAKE, FAKE, 0, None) == E_NULL
    assert lib.ic3_trace_comm_step(ctypes.byref(io), ctypes.byref(cm), None, FAKE, FAKE, FAKE, 0, None) == E_NULL
    _comm_refusals(_lib, call, io, cm)
    assert call(h=None) == E_NULL and call(g=None) == E_NULL and call(s=None) == E_NULL
    assert call(r=_copy(_lib.EvalTrace, tr, slots=None)) == E_NULL
    assert call(i=_copy(_lib.EvalStepIO, io, err=None)) == E_NULL
    for field in ("T", "K"):
        assert call(r=_copy(_lib.EvalTrace, tr, **{field: 0})) == E_RANGE, field
    # row t is written before policy step t: 0 <= t < T, no closing call
    assert call(t=-1) == E_RANGE and call(t=40) == E_RANGE


@pytest.mark.parametrize("tj", [False, True], ids=["pp", "tj"])
def test_message_map_step_checks_arguments(built_lib, tj):
    from ic3net_b200 import _lib
    lib = _lib.load()
    io, cm, _, keep = _io(_lib, tj)

    def call(i=io, c=cm, out=FAKE):
        return lib.ic3_message_map_step(ctypes.byref(i), ctypes.byref(c), out, None)
    assert call(out=None) == E_NULL
    assert lib.ic3_message_map_step(None, ctypes.byref(cm), FAKE, None) == E_NULL
    assert lib.ic3_message_map_step(ctypes.byref(io), None, FAKE, None) == E_NULL
    _comm_refusals(_lib, call, io, cm)


@pytest.mark.parametrize("tj", [False, True], ids=["pp", "tj"])
def test_message_map_blocks_and_means(tj):
    """Recorder._message_map splits the int64 sums by key row, scales them by 2^-32 and divides by the open senders
    (sent) and the comm map's visits (received), NaN where the count is 0."""
    from ic3net_b200.eval_trace import Recorder
    rec = object.__new__(Recorder)
    P, S, H = 6, 4, 16
    rec.npos, rec.max_steps, rec.H, rec.is_tj = P, S, H, tj
    R = rec.msg_rows = P + S + (0 if tj else 2)
    rng = np.random.default_rng(0)
    sent, recv = rng.integers(-2 ** 40, 2 ** 40, (R, H)), rng.integers(-2 ** 40, 2 ** 40, (R, H))
    senders = rng.integers(0, 3, R)
    visits = senders + rng.integers(0, 2, R)
    cmap = dict(visits=visits[:P], visits_t=visits[P:P + S])
    if not tj:
        cmap["visits_reached"] = visits[P + S:]
    out = rec._message_map(np.concatenate([sent.ravel(), recv.ravel(), senders]).astype(np.int64), cmap)
    assert out["msg_scale"] == 2.0 ** -32
    parts = [("", slice(0, P)), ("_t", slice(P, P + S))] + ([] if tj else [("_reached", slice(P + S, R))])
    expect = {"msg_scale"}
    for suffix, rows in parts:
        expect |= {k + suffix for k in ("msg_sent", "msg_recv", "msg_senders", "msg_sent_mean", "msg_recv_mean")}
        assert out["msg_sent" + suffix].dtype == np.int64
        assert np.array_equal(out["msg_sent" + suffix], sent[rows])
        assert np.array_equal(out["msg_recv" + suffix], recv[rows])
        assert np.array_equal(out["msg_senders" + suffix], senders[rows])
        for key, tot, n in (("msg_sent_mean", sent[rows], senders[rows]), ("msg_recv_mean", recv[rows], visits[rows])):
            m = out[key + suffix]
            assert np.isnan(m[n == 0]).all()
            assert np.array_equal(m[n > 0], tot[n > 0] * 2.0 ** -32 / n[n > 0, None]), key
    assert set(out) == expect
