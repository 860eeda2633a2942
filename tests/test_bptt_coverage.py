"""CPU tests of which policy configurations the BPTT kernels cover: ic3_bptt_workspace_bytes is > 0 exactly for them and
0 for everything else (Trainer asks it to choose grad_impl 'kernels'); no device work."""
import ctypes as C

import pytest

D, V = 20, 1                   # predator-prey 20 x 20, vision 1: 400 positions + 19 pattern columns
TJ_H = TJ_W = 8                # traffic junction 8 x 8, vision 1: 64 positions + 13 pattern columns


def heads(*dims):
    from ic3net_b200 import _lib
    return (C.c_int32 * _lib.MAX_HEADS)(*(list(dims) + [0] * (_lib.MAX_HEADS - len(dims))))


def lstm(**kw):
    """The recurrent LSTM CommNet / IC3Net on predator-prey (one pass, soft communication)."""
    from ic3net_b200 import _lib
    W = 2 * V + 1
    pol = dict(B=8, N=10, H=128, O=W * W * (D * D + 4), nheads=1, head_dim=heads(5), hard_attn=0, comm_avg=1,
               comm_mask_zero=0, env_id0=0, seed=1, obs_off=0, obs_vocab=D * D + 4, obs_ncount=2, cell=_lib.CELL_LSTM,
               passes=1, x_tanh=0, h_from_x=0)
    pol.update(kw)
    return pol


def tanh_rnn(**kw):
    """The tanh recurrence without communication (models.RNN with rnn_type 'MLP': the IC / IRIC baselines)."""
    from ic3net_b200 import _lib
    return lstm(**dict(dict(cell=_lib.CELL_TANH, comm_mask_zero=1), **kw))


def nbytes(pol, dim=D, vision=V, tj=False):
    from ic3net_b200 import _lib
    lib = _lib.load()
    cfg = _lib.PolicyCfg(**pol)
    if tj:
        vocab = TJ_H * TJ_W + 3
        env = _lib.TJCfg(B=pol["B"], N=pol["N"], vision=vision, h=TJ_H, w=TJ_W, G=4, P=3, Lmax=16,
                         outside_cls=vocab - 3, car_cls=vocab - 1, vocab=vocab, npath=12, env_id0=0, seed=1)
        plan = _lib.BpttPlan(cfg=C.pointer(cfg), w=None, pp_env=None, tj_env=C.pointer(env), x_table=None,
                             value_coeff=0.01, entr=0.0, workspace=None)
    else:
        env = _lib.PPCfg(B=pol["B"], N=pol["N"], dim=dim, vision=vision, mode=0, naction=5, env_id0=0, seed=1)
        plan = _lib.BpttPlan(cfg=C.pointer(cfg), w=None, pp_env=C.pointer(env), tj_env=None, x_table=None,
                             value_coeff=0.01, entr=0.0, workspace=None)
    return int(lib.ic3_bptt_workspace_bytes(C.byref(plan)))


def tj_layout(pol):
    vocab = TJ_H * TJ_W + 3
    return dict(pol, O=2 + 9 * vocab, obs_off=2, obs_vocab=vocab, obs_ncount=1)


# share_weights is no field of ic3_policy_cfg (the passes' weight and gradient pointers alias), so the pass counts
# below cover it
@pytest.mark.parametrize("kw", [dict(passes=1), dict(passes=2), dict(passes=3), dict(passes=4),
                                dict(hard_attn=1, nheads=2, head_dim=heads(5, 2)), dict(comm_avg=0)])
def test_lstm_policies_are_covered(kw):
    assert nbytes(lstm(**kw)) > 0


def test_tanh_rnn_is_covered_on_both_environments():
    assert nbytes(tanh_rnn()) > 0
    assert nbytes(tj_layout(tanh_rnn()), tj=True) > 0


@pytest.mark.parametrize("kw", [dict(H=64), dict(passes=5), dict(x_tanh=1), dict(h_from_x=1),
                                dict(nheads=2, head_dim=heads(5, 3))])                     # 9 outputs
def test_lstm_outside_the_kernels_gets_zero_bytes(kw):
    assert nbytes(lstm(**kw)) == 0


@pytest.mark.parametrize("kw", [dict(comm_mask_zero=0), dict(hard_attn=1), dict(passes=2)])
def test_tanh_cell_with_communication_or_passes_gets_zero_bytes(kw):
    assert nbytes(tanh_rnn(**kw)) == 0


def test_geometry_limits():
    # vision 3: a 7 x 7 window
    assert nbytes(lstm(O=49 * (D * D + 4)), vision=3) == 0
    # predator-prey dim 23: 529 positions + 19 pattern columns, 560 after padding, beyond 512
    assert nbytes(lstm(O=9 * (23 * 23 + 4), obs_vocab=23 * 23 + 4), dim=23) == 0


def test_observation_layout_hint_is_required():
    assert nbytes(lstm(obs_vocab=0, obs_ncount=0)) == 0                 # no layout hint
    assert nbytes(lstm(obs_ncount=1)) == 0                              # a hint that is not predator-prey's
    assert nbytes(tanh_rnn(obs_vocab=0, obs_ncount=0)) == 0
    assert nbytes(dict(tj_layout(tanh_rnn()), obs_ncount=2), tj=True) == 0
    assert nbytes(tanh_rnn(obs_vocab=D * D + 5)) == 0
