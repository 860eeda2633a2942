"""CPU tests of the bounded observation writers (ic3_pp_obs_bounded / ic3_tj_obs_bounded): a bad call is refused by
the host-side checks with the same codes as ic3_pp_obs / ic3_tj_obs, before anything is launched."""
import ctypes

E_NULL, E_RANGE = -1, -2
FAKE = 0x1000                      # never dereferenced: validation fails first


def _pp(_lib):
    env = _lib.PPCfg(B=4, N=3, dim=5, vision=1, mode=0, naction=5, env_id0=0, enemy_comm=0, seed=1)
    st = _lib.PPState(loc=FAKE, reached=FAKE, done=FAKE, success=FAKE, episode=FAKE, tick=FAKE)
    return env, st


def _tj(_lib):
    V = 14
    env = _lib.TJCfg(B=4, N=3, vision=1, h=14, w=14, G=4, P=3, Lmax=20, outside_cls=V - 3, car_cls=V - 1, vocab=V,
                     npath=12, spawn_thr=0, env_id0=0, seed=1, grid=FAKE, route_len=FAKE, route_cells=FAKE)
    st = _lib.TJState(loc=FAKE, alive=FAKE, wait=FAKE, route_id=FAKE, route_pos=FAKE, last_act=FAKE, completed=FAKE,
                      cars_in_sys=FAKE, has_failed=FAKE, tick=FAKE)
    return env, st


def test_pp_obs_bounded_checks_arguments(built_lib):
    from ic3net_b200 import _lib
    lib = _lib.load()
    env, st = _pp(_lib)
    for fn in (lib.ic3_pp_obs, lib.ic3_pp_obs_bounded):
        call = lambda e=env, s=st, obs=FAKE: fn(ctypes.byref(e), ctypes.byref(s), obs, None)
        assert call(obs=None) == E_NULL
        assert call(s=_lib.PPState()) == E_NULL
        for field, bad in (("B", 0), ("N", 32), ("dim", 0), ("vision", 8), ("mode", 3), ("naction", 3)):
            ec = _lib.PPCfg.from_buffer_copy(env)
            setattr(ec, field, bad)
            assert call(e=ec) == E_RANGE, (fn, field)


def test_tj_obs_bounded_checks_arguments(built_lib):
    from ic3net_b200 import _lib
    lib = _lib.load()
    env, st = _tj(_lib)
    for fn in (lib.ic3_tj_obs, lib.ic3_tj_obs_bounded):
        call = lambda e=env, s=st, obs=FAKE: fn(ctypes.byref(e), ctypes.byref(s), obs, None)
        assert call(obs=None) == E_NULL
        assert call(s=_lib.TJState()) == E_NULL
        ec = _lib.TJCfg.from_buffer_copy(env)
        ec.grid = None
        assert call(e=ec) == E_NULL
        for field, bad in (("B", 0), ("N", 33), ("vision", 8), ("npath", 1), ("vocab", 0)):
            ec = _lib.TJCfg.from_buffer_copy(env)
            setattr(ec, field, bad)
            assert call(e=ec) == E_RANGE, (fn, field)
