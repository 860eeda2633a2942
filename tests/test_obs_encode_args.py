"""CPU tests of the fused observation + encoder entry points (ic3_pp_obs_encode / ic3_tj_obs_encode): a bad call is
refused by the host-side checks with the same codes as the index-form encoders, before anything is launched."""
import ctypes

E_NULL, E_RANGE, E_UNSUPPORTED = -1, -2, -3
FAKE = 0x1000                      # never dereferenced: validation fails first


def _policy(_lib, **kw):
    hd = (ctypes.c_int32 * _lib.MAX_HEADS)(5, 2, 0, 0)
    d = dict(B=4, N=3, H=128, O=9 * 29, nheads=2, head_dim=hd, hard_attn=1, comm_avg=1, comm_mask_zero=0, env_id0=0,
             seed=1, obs_off=0, obs_vocab=0, obs_ncount=0, cell=_lib.CELL_LSTM, passes=1, x_tanh=0, h_from_x=0)
    d.update(kw)
    return _lib.PolicyCfg(**d)


def _packed(_lib):
    return _lib.PolicyPacked(enc_wT=FAKE, enc_b=FAKE, c_wT=FAKE, c_b=FAKE, lstm_wT=FAKE, lstm_b=FAKE, head_w=FAKE,
                             head_b=FAKE)


def test_pp_obs_encode_checks_arguments(built_lib):
    from ic3net_b200 import _lib
    lib = _lib.load()
    env = _lib.PPCfg(B=4, N=3, dim=5, vision=1, mode=0, naction=5, env_id0=0, enemy_comm=0, seed=1)   # O = 9 * 29
    st = _lib.PPState(loc=FAKE, reached=FAKE, done=FAKE, success=FAKE, episode=FAKE, tick=FAKE)
    w = _packed(_lib)
    call = lambda e=env, s=st, c=None, pk=w, obs=FAKE, x=FAKE: lib.ic3_pp_obs_encode(
        ctypes.byref(e), ctypes.byref(s), ctypes.byref(c if c is not None else _policy(_lib)), ctypes.byref(pk), obs, x,
        None)
    assert call(obs=None) == E_NULL and call(x=None) == E_NULL
    assert call(s=_lib.PPState()) == E_NULL
    assert call(pk=_lib.PolicyPacked()) == E_NULL
    assert call(c=_policy(_lib, H=100)) == E_UNSUPPORTED
    assert call(c=_policy(_lib, B=5)) == E_RANGE                               # B of env and policy differ
    assert call(c=_policy(_lib, N=4)) == E_RANGE                               # rows per env: N (+ prey with enemy_comm)
    assert call(c=_policy(_lib, O=9 * 29 + 1)) == E_RANGE                      # not the env's observation size
    assert call(c=_policy(_lib, obs_vocab=28, obs_ncount=2)) == E_RANGE        # layout hint of another env
    ec =_lib.PPCfg.from_buffer_copy(env)
    ec.mode = 3
    assert call(e=ec) == E_RANGE


def test_tj_obs_encode_checks_arguments(built_lib):
    from ic3net_b200 import _lib
    lib = _lib.load()
    V = 14
    env = _lib.TJCfg(B=4, N=3, vision=1, h=14, w=14, G=4, P=3, Lmax=20, outside_cls=V - 3, car_cls=V - 1, vocab=V,
                     npath=12, spawn_thr=0, env_id0=0, seed=1, grid=FAKE, route_len=FAKE, route_cells=FAKE)
    st = _lib.TJState(loc=FAKE, alive=FAKE, wait=FAKE, route_id=FAKE, route_pos=FAKE, last_act=FAKE, completed=FAKE,
                      cars_in_sys=FAKE, has_failed=FAKE, tick=FAKE)
    w = _packed(_lib)
    O = 2 + 9 * V
    call = lambda e=env, s=st, c=None, obs=FAKE, x=FAKE: lib.ic3_tj_obs_encode(
        ctypes.byref(e), ctypes.byref(s), ctypes.byref(c if c is not None else _policy(_lib, O=O)), ctypes.byref(w), obs,
        x, None)
    assert call(obs=None) == E_NULL and call(x=None) == E_NULL
    assert call(s=_lib.TJState()) == E_NULL
    assert call(c=_policy(_lib, O=O, H=96)) == E_UNSUPPORTED
    assert call(c=_policy(_lib, O=O, B=3)) == E_RANGE
    assert call(c=_policy(_lib, O=O, N=2)) == E_RANGE
    assert call(c=_policy(_lib, O=O - 1)) == E_RANGE
    assert call(c=_policy(_lib, O=O, obs_off=0, obs_vocab=V, obs_ncount=1)) == E_RANGE   # TJ hint has obs_off = 2
