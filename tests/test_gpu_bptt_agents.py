"""The BPTT kernels (csrc/bptt_tc.cu) at every kind of agent count from 1 to 32, against the float64 yardsticks of the
other BPTT tests, and the two one-lane-per-agent kernels on the same gradient path (ic3_returns_scan, ic3_stat_reduce)
at their lane limits.

Several paths of the backward depend on the agent count N: the operand preparation's per-environment sums hold
PREP_ROWS / N + 2 environments (66 at N = 1, 4 at N = 31) and environments straddle its 64-row CTAs and the 128-row
tiles in patterns N alone decides; the comm kernel (one warp per environment, a loop over N) has its own branch for
N < 2 and for comm_mask_zero; the heads, gates and tanh kernels read per-environment masks at row / N.  The cases
below reach N = 1, a full warp of 32 agents (traffic junction with 32 cars; predator-prey with 31 predators and the
communicating prey), and N that straddle both row blocks; each asserts the geometry and the record events it is there
for, so a later change of B or of the episode lengths cannot silently lose an edge.

Bars: the gradient bar of tests/gpu_harness.py: per tensor 1e-4 of
its largest entry, the encoder weight also per column, the action heads also 2^-20 of their sum of |terms|.  Returns:
2.5e-7 max(1, |ref|), two float32 ulps (the kernel sums in float64 and rounds once; the order of its sum over agents can
move that rounding by one ulp).  Statistics: counts and the err word exact, sums within 1e-12 of their sum of |terms|."""
import numpy as np
import pytest
import torch

from bptt_ref import heads_abs_sums, trainer_reference
from gpu_harness import (OPT_IN, TOL, assert_within_bar as within_bar, bar_errors, events, grads_of,
                         lstm_trainer as make_trainer, one_step, passes_trainer, pattern_columns,
                         rnn_records_reference, rnn_trainer, sweep_batch, trainer_within_bar, window_vs_full)
from helpers import load_golden
from passes_oracle import records_reference

pytestmark = pytest.mark.gpu

PP, PP_ENEMY, TJ = "grad_pp_hard_ic3net_h128", "grad_pp_enemy_ic3net_h128", "grad_tj_hard_ic3net_h128"
RNN_PP, RNN_TJ = "gradrnn_pp_hard_ic", "gradrnn_tj_iric"
B = 37                                  # slots: B * N is never a multiple of 128 below, so the last tile is ragged
SHORT = dict(batch_size=14, max_steps=10)
ENEMY_32 = dict(dim=6)                  # 31 predators and the prey need more than the fixture's 5 x 5 cells


def agents(name, N):
    """Fixture overrides for N agent rows per env: traffic junction N cars; predator-prey N predators, or N - 1
    predators and the communicating prey (--enemy_comm)."""
    a = load_golden(name)[0]["args"]
    if a["env_name"] == "traffic_junction":
        return dict(nagents=N)
    enemy = int(a["enemy_comm"])
    return dict(nfriendly=N - enemy, nagents=N)


def straddles(Bn, N, rows):
    """Does some env's row range [b N, b N + N) cross a multiple of ``rows``?"""
    first = np.arange(Bn, dtype=np.int64) * N
    return bool((first // rows != (first + N - 1) // rows).any())


def geometry(tr):
    Bn, N = tr.env.env.nenvs, tr.args.nagents
    R = Bn * N
    return dict(N=N, R=R, tiles=-(-R // 128), mod128=128 % N, prep64=straddles(Bn, N, 64), tile128=straddles(Bn, N, 128))


def assert_geometry(tr, N, split):
    """N agent rows, a ragged last tile, and envs straddling the 64-row prep CTAs and the 128-row tiles iff ``split``
    (which 64 % N == 0 rules out)."""
    g = geometry(tr)
    assert g["N"] == N and g["R"] % 128 != 0, g
    assert g["prep64"] == split and g["tile128"] == split, g
    assert split == (64 % N != 0), g
    return g


def assert_events(tr):
    """Episode starts inside the batch and detach cuts; halted slots in predator-prey, dead and live cars in traffic
    junction."""
    ev = events(tr)
    assert ev["fresh"] > 0, ev
    if tr.args.detach_gap <= tr.args.max_steps:
        assert ev["cut"] > 0, ev
    if tr.is_tj:
        alive = tr._buf["s_tjalive"][:tr._buf["T"]]
        ev["dead"] = int((alive == 0).sum())
        assert 0 < ev["dead"] < alive.numel(), ev
    else:
        assert ev["halted"] > 0, ev
    return ev


def assert_drop_last_fails(tr, got, gloss, ref, rloss, label):
    """The bar is sensitive: the reference without the last env slot fails it."""
    Bn = tr.env.env.nenvs
    last, _ = trainer_reference(tr, slots=(Bn - 1, Bn))
    dropped = {k: ref[k] - last[k] for k in ref}
    derrs = bar_errors(got, dropped, heads_abs_sums(tr))
    print("%s without the last slot: %s" % (label, " ".join("%s %.1e" % kv for kv in derrs.items())))
    assert any(v > TOL for v in derrs.values()), derrs


# ---------------------------------------------------------------------------------------------------- IC3Net, 1 pass

ONE_PASS = {
    # id: (fixture, N, envs straddle the 64-row prep CTAs / 128-row tiles, extra overrides)
    "pp-1": (PP, 1, False, {}),
    "pp-2": (PP, 2, False, {}),
    "pp-7": (PP, 7, True, {}),
    "pp-11": (PP, 11, True, {}),
    "pp-31": (PP, 31, True, {}),
    "pp-enemy-1+1": (PP_ENEMY, 2, False, {}),
    "pp-enemy-31+1": (PP_ENEMY, 32, False, ENEMY_32),
    "tj-2": (TJ, 2, False, {}),
    "tj-13": (TJ, 13, True, {}),
    "tj-32": (TJ, 32, False, {}),
    "tj-32-comm-mask-zero": (TJ, 32, False, dict(comm_mask_zero=True)),
}
SENSITIVE = ("pp-1", "tj-32")


@pytest.mark.parametrize("case", list(ONE_PASS))
def test_one_pass(case):
    name, N, split, over = ONE_PASS[case]
    tr = make_trainer(name, B, seed=77, id0=3, **dict(agents(name, N), **SHORT, **over))
    assert tr.grad_kernels
    g = assert_geometry(tr, N, split)
    tr.run_batch(0)
    ev = assert_events(tr)
    got, gloss = grads_of(tr)
    ref, rloss = trainer_reference(tr)
    label = "%s %s %s" % (case, g, ev)
    trainer_within_bar(tr, got, gloss, ref, rloss, label)
    if case in SENSITIVE:
        assert_drop_last_fails(tr, got, gloss, ref, rloss, label)


@pytest.mark.parametrize("case", ["R<64", "dgrad-2-tiles"])
def test_one_agent_row_thresholds(case):
    """N = 1: the most tiles and prep CTAs per env of any geometry.  Fewer rows than one prep CTA, and more tiles than
    SMs (dgrad CTAs with two tiles: about 128 SMs + 1 one-agent envs)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    probe = make_trainer(PP, 1, **agents(PP, 1))
    Bn = sweep_batch(case, sms, 1, pattern_columns(probe))
    tr = make_trainer(PP, Bn, seed=77, id0=3, **dict(agents(PP, 1), **SHORT))
    g = assert_geometry(tr, 1, False)
    assert (g["R"] < 64) if case == "R<64" else (g["tiles"] > sms and g["R"] == 128 * sms + 1), (g, sms)
    tr.run_batch(0)
    ev = assert_events(tr)
    got, gloss = grads_of(tr)
    ref, rloss = trainer_reference(tr)
    trainer_within_bar(tr, got, gloss, ref, rloss, "%s B=%d SMs=%d %s %s" % (case, Bn, sms, g, ev))


# ---------------------------------------------------------------------------------------------------- comm passes

MULTI_PASS = {
    # id: (fixture, N, split, passes, share_weights, extra overrides)
    "pp-1-2pass": (PP, 1, False, 2, False, {}),
    "pp-7-2pass": (PP, 7, True, 2, False, {}),
    "pp-31-2pass": (PP, 31, True, 2, False, {}),
    "tj-2-commnet-3pass-sum": (TJ, 2, False, 3, True, dict(comm_mode="sum", hard_attn=False)),
    "tj-32-commnet-3pass-sum": (TJ, 32, False, 3, True, dict(comm_mode="sum", hard_attn=False)),
}


@pytest.mark.parametrize("case", list(MULTI_PASS))
def test_comm_passes(case):
    """IC3Net with 2 passes, and CommNet with 3 passes of one shared C module summing the messages (comm_mode sum)."""
    name, N, split, P, share, over = MULTI_PASS[case]
    tr = passes_trainer(name, B, seed=77, id0=3, comm_passes=P, share_weights=share,
                        **dict(agents(name, N), **SHORT, **over))
    assert tr.grad_kernels
    g = assert_geometry(tr, N, split)
    tr.run_batch(0)
    ev = assert_events(tr)
    got, gloss = grads_of(tr)
    ref, rloss = records_reference(tr)
    trainer_within_bar(tr, got, gloss, ref, rloss, "%s %s %s" % (case, g, ev))


# ---------------------------------------------------------------------------------------------------- IC / IRIC

RNN_CASES = {
    "ic-pp-1": (RNN_PP, 1, False),
    "ic-pp-31": (RNN_PP, 31, True),
    "iric-tj-32": (RNN_TJ, 32, False),
}


@pytest.mark.parametrize("case", list(RNN_CASES))
def test_tanh_rnn(case):
    name, N, split = RNN_CASES[case]
    tr = rnn_trainer(name, B, seed=77, id0=3, **dict(agents(name, N), **SHORT))
    assert tr.grad_kernels and tr.grad_impl == "kernels"
    g = assert_geometry(tr, N, split)
    tr.run_batch(0)
    ev = assert_events(tr)
    got, gloss = grads_of(tr)
    ref, rloss = rnn_records_reference(tr)
    trainer_within_bar(tr, got, gloss, ref, rloss, "%s %s %s" % (case, g, ev))


# ---------------------------------------------------------------------------------------------------- forward_grad

FORWARD_GRAD = {
    "pp-1": (PP, 1, 1, {}),
    "pp-1-2pass": (PP, 1, 2, {}),
    "pp-enemy-31+1": (PP_ENEMY, 32, 1, ENEMY_32),
    "tj-32": (TJ, 32, 1, {}),
}


@pytest.mark.parametrize("case", list(FORWARD_GRAD))
def test_forward_grad_one_step(case):
    """ic3_policy_step_backward (CommNetMLP.forward with forward_grad='kernels'): the gradients of the weights and of
    (h, c) under random upstream gradients against float64 autograd of the step."""
    name, N, P, over = FORWARD_GRAD[case]
    tr = passes_trainer(name, B, seed=5, id0=0, comm_passes=P, **dict(OPT_IN, **agents(name, N), **SHORT, **over))
    assert tr.args.nagents == N
    tr.rollout(tr.args.max_steps + 4, 0)
    b = tr._buf
    assert int(b["s_fresh"][1:].sum()) > 0
    t = tr.args.max_steps - 2
    if tr.is_tj:
        assert 0 < int(b["s_tjalive"][t].sum()) < b["s_tjalive"][t].numel()
    got, ref, sums = one_step(tr, t)
    assert "h" in got and "c" in got
    within_bar(got, ref, sums, "%s B=%d N=%d passes=%d" % (case, B, N, P))


# ---------------------------------------------------------------------------------------------------- windows

@pytest.mark.parametrize("name,N", [(PP, 1), (TJ, 32)])
def test_windowed_records_are_bit_identical(name, N):
    _, tf = window_vs_full(name, B, 4, **dict(agents(name, N), **SHORT))
    assert tf.args.nagents == N


# ---------------------------------------------------------------------------------------------------- returns scan

def returns_f64(reward, emask, mini, gamma, mean_ratio):
    """oracle.grad.returns_np over every env slot at once: reward / mini [T, B, N], emask [T, B] -> [T, B, N]."""
    T = reward.shape[0]
    coop, ncoop = np.zeros(reward.shape[1:]), np.zeros(reward.shape[1:])
    ret = np.zeros(reward.shape)
    em = emask[..., None]
    for i in reversed(range(T)):
        coop = reward[i] + gamma * coop * em[i]
        ncoop = reward[i] + gamma * ncoop * em[i] * mini[i]
        ret[i] = mean_ratio * coop.mean(-1, keepdims=True) + (1 - mean_ratio) * ncoop
    return ret


@pytest.mark.parametrize("Bn", [1, 3, 4097])
@pytest.mark.parametrize("N", [1, 31, 32])
def test_returns_scan_lane_limits(N, Bn):
    """T = 579 (predator-prey hard at batch_size 500); 4097 slots leave the last block of 4 warps with one."""
    from ic3net_b200 import _lib
    from oracle import grad as ograd
    T = 579
    rs = np.random.RandomState(N * 10007 + Bn)
    reward = rs.randn(T, Bn, N).astype(np.float32)
    emask = (rs.rand(T, Bn) > 0.05).astype(np.uint8)
    mini = (rs.rand(T, Bn, N) > 0.1).astype(np.uint8)
    assert (emask == 0).any() and (mini == 0).any()
    r, e, m = (torch.tensor(x, device="cuda") for x in (reward, emask, mini))
    out = torch.empty(T, Bn, N, device="cuda")
    r64, e64, m64 = reward.astype(np.float64), emask.astype(np.float64), mini.astype(np.float64)
    worst = 0.0
    for gamma in (1.0, 0.99):
        for mr in (0.0, 1.0, 0.4):
            g32, mr32 = np.float32(gamma).item(), np.float32(mr).item()     # what the kernel's float arguments hold
            out.fill_(np.nan)
            _lib.check(_lib.load().ic3_returns_scan(T, Bn, N, gamma, mr, r.data_ptr(), e.data_ptr(), m.data_ptr(),
                                                    out.data_ptr(), _lib.stream()))
            got = out.cpu().numpy().astype(np.float64)
            want = returns_f64(r64, e64, m64, g32, mr32)
            for b in sorted({0, Bn // 2, Bn - 1}):        # the batched form is returns_np slot by slot
                one = ograd.returns_np(r64[:, b], np.repeat(e64[:, b, None], N, 1), m64[:, b], g32, mr32)
                assert np.allclose(want[:, b], one, rtol=1e-13, atol=1e-13), b
            err = np.abs(got - want) / np.maximum(1.0, np.abs(want))
            worst = max(worst, float(err.max()))
            assert err.max() <= 2.5e-7, (gamma, mr, float(err.max()), np.unravel_index(err.argmax(), err.shape))
    print("returns N=%d B=%d: worst %.2e of max(1, |ref|)" % (N, Bn, worst))


# ---------------------------------------------------------------------------------------------------- stat reduce

GUARD = 8


@pytest.mark.parametrize("with_err", [False, True])
@pytest.mark.parametrize("with_comm", [False, True])
@pytest.mark.parametrize("N", [1, 32])
@pytest.mark.parametrize("Bn", [1, 7, 511, 512, 513, 8192])
def test_stat_reduce(Bn, N, with_comm, with_err):
    """One warp per slot, lane = agent; the grid grows with B up to 512 slots and is 64 blocks from there."""
    from ic3net_b200 import _lib
    rs = np.random.RandomState(Bn * 64 + N)
    episodes = rs.randint(0, 40, Bn).astype(np.int32)
    steps = rs.randint(0, 600, Bn).astype(np.int32)
    success = rs.randint(0, 3, Bn).astype(np.int32)
    reward = (rs.randn(Bn, N) * 10).astype(np.float32)
    comm = rs.rand(Bn, N).astype(np.float32)
    err = np.array([0x105], dtype=np.int32)
    dev = {k: torch.tensor(v, device="cuda") for k, v in dict(episodes=episodes, steps=steps, success=success,
                                                              reward=reward, comm=comm, err=err).items()}
    n = 4 + 2 * N
    out = torch.full((n + GUARD,), -7.25, dtype=torch.float64, device="cuda")
    _lib.check(_lib.load().ic3_stat_reduce(Bn, N, dev["episodes"].data_ptr(), dev["steps"].data_ptr(),
                                           dev["success"].data_ptr(), dev["err"].data_ptr() if with_err else None,
                                           dev["reward"].data_ptr(), dev["comm"].data_ptr() if with_comm else None,
                                           out.data_ptr(), _lib.stream()))
    got = out.cpu().numpy()
    assert got[0] == episodes.sum() and got[1] == steps.sum() and got[2] == success.sum(), got[:4]
    assert got[3] == (0x105 if with_err else 0.0), got[3]
    for off, x in ((4, reward), (4 + N, comm if with_comm else np.zeros_like(comm))):
        x = x.astype(np.float64)
        want, scale = x.sum(0), np.abs(x).sum(0)
        assert (np.abs(got[off:off + N] - want) <= 1e-12 * scale).all(), (off, got[off:off + N] - want)
    assert (got[n:] == -7.25).all(), got[n:]
