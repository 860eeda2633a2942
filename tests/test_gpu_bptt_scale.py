"""The power-of-two scale of the BPTT kernels' fp16 hi/lo operands (csrc/bptt_tc.cu) when gradient magnitudes swing
across steps, env slots and comm passes.

Each backward unit writes its d-gates (LSTM) or dz (tanh) operand multiplied by s = 2^e, chosen on the device by
bptt_scale_kernel from an upper bound of the unit's largest element:
bound = (dhmax + hbound[q] + dcmax) * max(1, cmax / 4), with bound * s in (2^13, 2^14].  q is the parity of the unit:
two buffer sets, scales and head bounds alternate, and the look-ahead heads of step t - 1 run before step t.  An
fp16 hi part overflows above 65504, four times the target, so an underestimate of more than about 4x writes inf into
the image and the update would apply a NaN gradient.  At initialisation-scale weights and the fixtures' rewards the
bounds of neighbouring units round to nearly the same power of two, so a unit reading its neighbour's slot, or a
reduction that misses rows, stays within the bar; the cases here make such faults overflow:

  - step-to-step swings: gamma 0, the rewards of even (or odd) steps x1e4, or the first half x1e-4 and the second half
    x1e4, with detach_gap 1 (every step cut) and the fixture's; ragged last tiles; the one-stream schedule and window
    records bit-identical to the default; comm_passes 2 and 3 (shared, sum mode), where units alternate the parity
    inside a step; the IC tanh RNN on 'simt' and 'tc_tanh'; the full batch sizes;
  - one env slot dominating (x1e6 on alternate steps): at slot 0, straddling a 128-row tile, the last slot of a ragged
    tile, and the last slot at full size (the head-bound, dh and dc reductions cover every row);
  - head weights x1e-5 and x1e3 after the rollout, and one large entry in hidden unit 127 of an action head or the
    value head (the heads' per-output weight maximum);
  - saturated cells with |c| past 20, and cells whose f gate carries dc while the recurrent weights keep dh small (the
    cmax and dcmax terms);
  - ic3_bptt_begin_dev's max |c| against ic3_bptt_begin with the host maximum on crafted arrays (tail, misalignment,
    grid stride, past 2^31 elements);
  - ic3_policy_step_backward with upstream gradients x1e-6 and x1e4, and one spike in dh, dc or dvalue.

Perturbations enter the records or the weights between the rollout and compute_grad (rewards: the returns are computed
from them; head weights: the heads' backward starts from the recorded log-probs and values), so the kernels and the
float64 yardstick read the same inputs.  Bar: the gradient bar of tests/gpu_harness.py, every gradient entry
finite, the error word 0.  Each case asserts its own precondition in float64 so that it cannot pass vacuously."""
import ctypes as C

import pytest
import torch

from bptt_ref import returns_and_advantages, trainer_reference
from gpu_harness import (GAMMA0, OPT_IN, PP, SMALL, TJ, assert_within_bar, finite_and_clean, grads_of,
                         lstm_trainer as make_trainer, one_step, one_stream_schedule, passes_trainer,
                         rnn_records_reference, rnn_trainer, swing, trainer_within_bar)
from passes_oracle import records_reference as passes_reference

pytestmark = pytest.mark.gpu

FULL = {PP: 8192, TJ: 4096}


# ---------------------------------------------------------------------------------------------------- helpers

def dominate(tr, k, factor=1e6):
    """Scale the rewards of env slot k on odd steps: there its heads dominate every other slot's, and on even steps
    the d(h, c) it sends back dominates the step's own head bound."""
    r, T = tr._buf["reward"], tr._buf["T"]
    with torch.no_grad():
        r[1:T:2, k] *= factor
    _, adv = returns_and_advantages(tr)
    a = (adv.to(torch.float64) * tr._buf["ralive"][:T].to(torch.float64)).abs()[1:T:2]       # [T', B, N]
    mine = a[:, k].amax().item()
    others = torch.cat([a[:, :k], a[:, k + 1:]], 1).amax().item()
    assert mine >= 1e4 * others, (k, mine, others)


def check_lstm(tr, label, reference=trainer_reference):
    got, gloss = grads_of(tr)
    finite_and_clean(tr, got, label)
    ref, rloss = reference(tr)
    errs = trainer_within_bar(tr, got, gloss, ref, rloss, label)
    print("%s: worst error %.2e (bar 1e-4)" % (label, max(errs.values())))
    return got, gloss


def check_rnn(tr, label):
    got, gloss = grads_of(tr)
    finite_and_clean(tr, got, label)
    ref, rloss = rnn_records_reference(tr)
    trainer_within_bar(tr, got, gloss, ref, rloss, label)


def scale_heads(tr, factor):
    with torch.no_grad():
        for k, p in tr.policy_net.named_parameters():
            if k.endswith(".weight") and ("heads." in k or "value_head" in k):
                p.mul_(factor)


def gates(tr):
    """(i, f, g, o) slices of the LSTM's gate rows."""
    H = tr.args.hid_size
    return [slice(j * H, (j + 1) * H) for j in range(4)]


# ---------------------------------------------------------------------------------------------------- swings

@pytest.mark.parametrize("pattern", ["even", "odd", "block"])
@pytest.mark.parametrize("gap", ["1", "fixture"])
@pytest.mark.parametrize("name", [PP, TJ])
def test_step_swings(name, gap, pattern):
    """Neighbouring steps' bounds differ by 1e4: a unit reading the other parity's head bound, scale or inverse scale
    overflows in one of the two mirrored patterns.  detach_gap 1: every step's incoming d(h, c) is dropped."""
    over = dict(GAMMA0, **({"detach_gap": 1} if gap == "1" else {}))
    tr = make_trainer(name, SMALL[name], seed=41, id0=5, **over)
    tr.run_batch(0)
    ratio = swing(tr, pattern)
    check_lstm(tr, "%s B=%d detach_gap=%d %s (80%% of step ratios >= %.1e)" % (name, SMALL[name], tr.args.detach_gap,
                                                                              pattern, ratio))


def test_swings_one_stream_schedule_is_bit_identical(tmp_path):
    """Kernel gradients and losses of two swing batches (even steps of predator-prey, odd steps of traffic junction)."""
    one_stream_schedule(tmp_path, "gpu_harness", "swing_grads", more_than=2, timeout=900)


@pytest.mark.parametrize("name,pattern", [(PP, "odd"), (TJ, "even")])
def test_swings_window_records_are_bit_identical(name, pattern):
    """Window records (full records never fit): the recomputed (h, c) and the device max |c| of the rollout's per-step
    maxima give the same gradient bit for bit."""
    out = []
    for windows in (False, True):
        tr = make_trainer(name, SMALL[name], seed=41, id0=5, windows=windows, **GAMMA0)
        tr.run_batch(0)
        swing(tr, pattern)
        got, s = grads_of(tr)
        finite_and_clean(tr, got, name)
        out.append((tr.record_mode, got, s))
    (m0, g0, s0), (m1, g1, s1) = out
    assert m0 == "full" and m1 == "window"
    assert all(torch.equal(g0[k], g1[k]) for k in g0), [k for k in g0 if not torch.equal(g0[k], g1[k])]
    assert s0 == s1


@pytest.mark.parametrize("name,passes,share,over,pattern", [
    (PP, 2, False, {}, "even"),
    (PP, 2, False, {}, "odd"),
    (TJ, 3, True, dict(comm_mode="sum", hard_attn=False), "even"),
    (TJ, 3, True, dict(comm_mode="sum", hard_attn=False), "block"),
])
def test_swings_comm_passes(name, passes, share, over, pattern):
    """comm_passes > 1: the units (t, P-1) .. (t, 0) alternate the parity inside a step and nothing is launched ahead;
    the heads (last pass) and the recursion-only passes get bounds from different terms."""
    tr = passes_trainer(name, SMALL[name], seed=41, id0=5, comm_passes=passes, share_weights=share,
                        **dict(GAMMA0, **over))
    tr.run_batch(0)
    swing(tr, pattern)
    check_lstm(tr, "%s passes=%d share=%s %s %s" % (name, passes, share, over, pattern), passes_reference)


@pytest.mark.parametrize("pattern", ["even", "odd"])
@pytest.mark.parametrize("impl", ["simt", "tc_tanh"])
@pytest.mark.parametrize("name", [PP, TJ])
def test_swings_tanh_rnn(name, impl, pattern):
    """The IC tanh RNN: the dz operand takes the scale of its unit."""
    tr = rnn_trainer(name, SMALL[name], seed=41, id0=5, policy_impl=impl, **GAMMA0)
    tr.run_batch(0)
    swing(tr, pattern)
    check_rnn(tr, "IC %s B=%d %s %s" % (name, SMALL[name], impl, pattern))


@pytest.mark.parametrize("name,pattern", [(PP, "even"), (TJ, "odd")])
def test_swings_full_size(name, pattern):
    tr = make_trainer(name, FULL[name], seed=5, id0=0, **GAMMA0)
    tr.run_batch(0)
    swing(tr, pattern)
    check_lstm(tr, "%s B=%d %s" % (name, FULL[name], pattern))


# ---------------------------------------------------------------------------------------------------- one slot

def close_forget_gate(tr):
    """f ~ 3e-4 (bias -8, before the rollout): d c_{t-1} = d c_t f carries almost nothing back, so the d h a step
    sends back is the only large term of the next unit's bound and dhmax alone has to cover the dominating slot."""
    set_gate_bias(tr, f=-8.0)


@pytest.mark.parametrize("forget", ["open", "closed"])
@pytest.mark.parametrize("where", ["first", "straddles-tile", "last"])
def test_one_slot_dominates(where, forget):
    """Predator-prey, 10 agents: slot 12 holds rows 120..129 across the first tile boundary; slot 36 holds rows
    360..369 of the ragged last tile (370 rows)."""
    B = SMALL[PP]
    k = {"first": 0, "straddles-tile": 12, "last": B - 1}[where]
    tr = make_trainer(PP, B, seed=41, id0=5, **GAMMA0)
    N = tr.args.nagents
    assert where != "straddles-tile" or (k * N) // 128 != (k * N + N - 1) // 128
    if forget == "closed":
        close_forget_gate(tr)
    tr.run_batch(0)
    dominate(tr, k)
    check_lstm(tr, "PP B=%d slot %d dominates, forget gate %s" % (B, k, forget))


@pytest.mark.parametrize("forget", ["open", "closed"])
@pytest.mark.parametrize("name", [PP, TJ])
def test_last_slot_dominates_full_size(name, forget):
    B = FULL[name]
    tr = make_trainer(name, B, seed=5, id0=0, **GAMMA0)
    if forget == "closed":
        close_forget_gate(tr)
    tr.run_batch(0)
    dominate(tr, B - 1)
    check_lstm(tr, "%s B=%d last slot dominates, forget gate %s" % (name, B, forget))


# ---------------------------------------------------------------------------------------------------- head weights

@pytest.mark.parametrize("case", ["x1e-5", "x1e3", "action-unit-127", "value-unit-127"])
@pytest.mark.parametrize("name", [PP, TJ])
def test_head_weight_extremes(name, case):
    """After the rollout: every head weight scaled (both ends of the operand range), or one entry of hidden unit 127
    made 1e3 times the largest weight of its head (the heads' bound takes its maximum over every unit)."""
    tr = make_trainer(name, SMALL[name], seed=41, id0=5)
    tr.run_batch(0)
    net = tr.policy_net
    if case.startswith("x"):
        scale_heads(tr, float(case[1:]))
    else:
        w = net.heads[0].weight if case.startswith("action") else net.value_head.weight
        with torch.no_grad():
            big = 1e3 * float(w.abs().max())
            w[-1, 127] = -big if case.startswith("action") else big
        assert float(w[:, :64].abs().max()) * 1e2 < big and float(w[:, 64:127].abs().max()) * 1e2 < big
    check_lstm(tr, "%s heads %s" % (name, case))


# ---------------------------------------------------------------------------------------------------- cell state

def set_gate_bias(tr, **bias):
    """LSTM gate biases (bias_ih + bias_hh) of gates i, f, g, o set to constants, before the rollout."""
    sl = dict(zip("ifgo", gates(tr)))
    with torch.no_grad():
        for gname, v in bias.items():
            tr.policy_net.f_module.bias_ih[sl[gname]] = v
            tr.policy_net.f_module.bias_hh[sl[gname]] = 0.0


@pytest.mark.parametrize("pattern", ["even", "odd"])
@pytest.mark.parametrize("name", [PP, TJ])
def test_saturated_cells(name, pattern):
    """i, f, g saturated before the rollout: c grows by about 1 per step (|c| past 20), the bound's max(1, cmax / 4)
    factor is large and d c is carried through f ~ 1."""
    from ic3net_b200 import _lib
    tr = make_trainer(name, SMALL[name], seed=41, id0=5, max_steps=40, **GAMMA0)
    set_gate_bias(tr, i=6.0, f=6.0, g=3.0)
    tr.run_batch(0)
    assert int(tr._buf["err"].item()) & _lib.ERR_FP16_RANGE == 0
    T = tr._buf["T"]
    cmax = float(tr._buf["rec_c"][1:T + 1].abs().max())
    assert cmax >= 20.0, cmax
    swing(tr, pattern)
    check_lstm(tr, "%s saturated cells max|c| %.1f %s" % (name, cmax, pattern))


@pytest.mark.parametrize("name", [PP, TJ])
def test_cell_gradient_dominates(name):
    """f ~ 1 carries d c back undamped while the recurrent and comm weights (x1e-3) leave d h small: after a large step,
    the next unit's bound is almost all dcmax."""
    tr = make_trainer(name, SMALL[name], seed=41, id0=5, **GAMMA0)
    net = tr.policy_net
    with torch.no_grad():
        net.f_module.weight_hh.mul_(1e-3)
        for m in net.C_modules:
            m.weight.mul_(1e-3)
    set_gate_bias(tr, f=8.0)
    tr.run_batch(0)
    swing(tr, "even")
    T = tr._buf["T"]
    cmax = float(tr._buf["rec_c"][1:T + 1].abs().max())
    assert cmax < 16.0, cmax              # max(1, cmax / 4) stays small: dcmax is the bound's only large term
    check_lstm(tr, "%s d c dominates, max|c| %.1f" % (name, cmax))


# ---------------------------------------------------------------------------------------------------- device max |c|

def begin_workspaces(plan, c, n):
    """(host-begin workspace, device-begin workspace) bytes from zero, for the n floats at c (a float32 tensor view)."""
    from ic3net_b200 import _lib
    lib, s = _lib.load(), _lib.stream()
    ws = torch.zeros(int(lib.ic3_bptt_workspace_bytes(C.byref(plan))), dtype=torch.uint8, device="cuda")
    plan.workspace = ws.data_ptr()
    cmax = float(c[:n].abs().max())
    _lib.check(lib.ic3_bptt_begin(C.byref(plan), cmax, s))
    torch.cuda.synchronize()
    host = ws.clone()
    ws.zero_()
    _lib.check(lib.ic3_bptt_begin_dev(C.byref(plan), C.c_void_p(c.data_ptr()), n, s))
    torch.cuda.synchronize()
    return host, ws, cmax


def lstm_plan(passes):
    from ic3net_b200 import _lib
    tr = passes_trainer(PP, 5, seed=41, id0=5, comm_passes=passes)
    tr.run_batch(0)
    plan = tr._bptt_plan(tr._policy_cfg(), tr.policy_net.packed(), _lib.ptr(tr._encoder_table()))
    return tr, plan


def crafted(n, where, off, gen):
    """float32 device buffer with n values from offset off (floats) of its storage: |values| < 1, and the maximum
    (7.5, or -7.5 for 'negative') at `where`; 'zeros' all -0.0."""
    base = torch.empty(n + off + 4, device="cuda")
    c = base[off:off + n]
    if where == "zeros":
        c.fill_(-0.0)
        return c
    c.copy_(torch.rand(n, generator=gen, device="cuda") * 2 - 1)
    i = {"first": 0, "last": n - 1, "tail": n - 1 - (n % 4 > 1), "middle": n // 2, "negative": n // 3}[where]
    c[i] = -7.5 if where == "negative" else 7.5
    return c


@pytest.mark.parametrize("passes", [1, 3])
def test_device_cmax_matches_host_cmax(passes):
    """ic3_bptt_begin_dev leaves the workspace of ic3_bptt_begin given the host maximum: short arrays (the scalar tail
    alone), 4k + 3 floats, past one grid-stride pass, a pointer off by one float (no float4 path), the maximum first,
    last, in the tail, negative, and all -0.0."""
    _, plan = lstm_plan(passes)
    grid = 4 * torch.cuda.get_device_properties(0).multi_processor_count * 256 * 4    # floats per grid-stride pass
    gen = torch.Generator(device="cuda").manual_seed(3)
    cases = []
    for n in (1, 3, 5, 4 * 1001 + 3, 3 * grid + 7):
        for where in ("first", "last", "tail", "negative", "zeros"):
            for off in (0, 1):
                cases.append((n, where, off))
    cases.append((2 * grid, "middle", 0))
    for n, where, off in cases:
        c = crafted(n, where, off, gen)
        assert off == 0 or c.data_ptr() % 16 != 0
        host, dev, cmax = begin_workspaces(plan, c, n)
        assert cmax == (0.0 if where == "zeros" else 7.5)
        assert torch.equal(host, dev), (passes, n, where, off)
    print("device max |c|: %d arrays, P=%d, bit-identical workspaces" % (len(cases), passes))


def test_device_cmax_past_2_31_floats():
    """Full records at two comm passes reach about 6e9 floats: the device reduction indexes them in 64 bits."""
    n = (1 << 31) + 11
    need = (n + 64) * 4 + (1 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        msg = "needs %.1f GB free on the device, %.1f GB free" % (need / 1e9, free / 1e9)
        print("skipped: " + msg)
        pytest.skip(msg)
    _, plan = lstm_plan(1)
    base = torch.zeros(n + 8, device="cuda")
    for off, i in ((0, (1 << 31) + 9), (1, n - 1)):       # past 2^31 in the float4 loop; in the tail, misaligned
        c = base[off:off + n]
        c.zero_()
        c[i] = 3.25
        c[(1 << 30) + 1] = -2.0
        host, dev, cmax = begin_workspaces(plan, c, n)
        assert cmax == 3.25
        assert torch.equal(host, dev), (off, i)
    del base
    print("device max |c| over %d floats: bit-identical workspaces" % n)


# ---------------------------------------------------------------------------------------------------- upstream

@pytest.mark.parametrize("scale,spike", [(1e-6, None), (1e4, None), (1.0, "dh"), (1.0, "dc"), (1.0, "dvalue")])
def test_upstream_extremes(scale, spike):
    """ic3_policy_step_backward reduces the maxima of the caller's d h', d c' (and the heads' bound of d value) on the
    device; a spike of 1e5 in the last row and column of one of them must reach the bound."""
    tr = passes_trainer(PP, SMALL[PP], seed=5, id0=0, **OPT_IN)
    tr.rollout(tr.args.max_steps + 4, 0)
    got, ref, sums = one_step(tr, tr.args.max_steps - 2, scale=scale, spike=None if spike is None else (spike, 1e5))
    bad = [k for k, v in got.items() if not torch.isfinite(v).all()]
    assert not bad, bad
    errs = assert_within_bar(got, ref, sums, "upstream x%g spike %s" % (scale, spike))
    print("upstream x%g spike %s: worst error %.2e (bar 1e-4)" % (scale, spike, max(errs.values())))
