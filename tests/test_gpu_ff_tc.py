"""GPU tests of the non-recurrent tanh policies' tensor-core policy step (csrc/ff_tc.cu, policy_impl 'tc_ff': models.MLP and
CommNet / IC3Net without --recurrent).

Covered: every row of every step of a rollout with episode resets (and dead cars on traffic junction) at the full batch
sizes against a float64 step fed from the trainer's records; the reference's forward fixtures and every gradff_* gradient
fixture through grad_impl 'kernels_ff' with this forward; the kernels_ff re-run (ic3_policy_ff_states) against the
rollout's step bit for bit; the gradient against float64 at full size for 1, 2 and 4 passes with and without
share_weights, run to run and with halted slots; row counts around the 64-row tile and the persistent-grid thresholds;
agents per env from 1 to 32 (padding rows inside a tile, envs of different sizes); rows past R; sampling with explicit
draws against the SIMT path; the fp16 limits; CUDA-graph rollouts; the refusals; the command line.

Bar of the forward: |gpu - ref| <= 1e-5 * max(1, |ref|) on h', value and log-probs (DESIGN.md section 2), except
comm_mode sum with several passes (sum_tol): there S is up to N - 1 times an h, its fp16 hi/lo split and the tensor-core
accumulation carry a relative error a few times fp32's, and each pass multiplies the error of h by up to N - 1 through
the next S.  The bar there is 3e-6 (N - 1), at least 1e-5: 3 passes measured 1.1e-5 at N = 10, 1.8e-5 with the 20
traffic-junction agents, 5.8e-5 at N = 32."""
import argparse
import ctypes as C

import numpy as np
import pytest
import torch

from gpu_harness import (MARGIN, PP, ROW_TOL, TJ, assert_close, close, compare_rows, ff_chunk_sizes_and_determinism,
                         ff_direct_step, ff_full_size, ff_gradient_arrays, ff_halted_slots_contribute_nothing, ff_net,
                         ff_pinned_oracle, ff_step_f64, ff_trainer, gated_mean, gates_f64, rollout_and_grad, sum_tol,
                         variant_net)
from helpers import golden_names, load_golden
from policy_ref import inverse_cdf

pytestmark = pytest.mark.gpu

TILE = 64                   # rows per CTA tile of ff_tc_kernel


def make_trainer(name, B, family, **kw):
    kw.setdefault("policy_impl", "tc_ff")
    tr = ff_trainer(name, B, family, **kw)
    assert tr.policy_net.policy_impl == kw["policy_impl"]
    return tr


def compare(label, got, ref, worst=None, tol=ROW_TOL):
    compare_rows(label, got, ref, worst, tol)


# ---------------------------------------------------------------------------------------------------- direct steps

def twin_nets(N, heads, family="ic3net", wseed=3, **kw):
    tc, simt = ff_net(N, heads, "tc_ff", family, wseed=wseed, **kw), ff_net(N, heads, "simt", family, wseed=wseed, **kw)
    simt.load_state_dict(tc.state_dict())
    return tc, simt


def inputs(B, N, seed, scale=1.5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B * N, 128, generator=g, device="cuda") * scale
    comm = torch.randint(0, 2, (B, N), generator=g, device="cuda", dtype=torch.uint8)
    alive = (torch.rand(B, N, generator=g, device="cuda") < 0.8).to(torch.uint8)
    fresh = (torch.arange(B, device="cuda") % 5 == 0).to(torch.uint8)
    return x, comm, alive, fresh


def outputs(R, heads, extra=0):
    nan = lambda *s: torch.full(s, 0x7FC0DEAD, dtype=torch.int32, device="cuda").view(torch.float32)
    return dict(h=nan(R + extra, 128), value=nan(R + extra), logp=nan(R + extra, sum(heads)),
                action=torch.full((R + extra, len(heads)), -7, dtype=torch.int32, device="cuda"))


def record_inputs(tr, t):
    """x (index encoder on the recorded env state) and the masks entering lock-step t of the trainer's records."""
    from ic3net_b200 import _lib
    b, e, net = tr._buf, tr.env.env, tr.policy_net
    lib = _lib.load()
    B, N = e.nenvs, tr.args.nagents
    cfg, w = net.policy_cfg(B), net.packed()
    ecfg, est = tr._record_state(t)
    x = torch.empty(B * N, 128, device="cuda")
    enc = lib.ic3_tj_encoder_index if tr.is_tj else lib.ic3_pp_encoder_index
    _lib.check(enc(C.byref(ecfg), C.byref(est), C.byref(cfg), C.byref(w), x.data_ptr(), _lib.stream()))
    hard = bool(tr.args.hard_attn) and bool(tr.args.commnet)
    return dict(x=x, comm=b["s_comm"][t] if hard else None, alive=b["s_alive"][t], fresh=b["s_fresh"][t])


# ---------------------------------------------------------------------------------------------------- 1. full size

FULL = [(PP, 8192, "mlp", {}), (PP, 8192, "ic3net", {}), (PP, 8192, "commnet", dict(comm_passes=2)),
        (TJ, 4096, "ic3net", {}), (TJ, 4096, "commnet", dict(comm_passes=3, share_weights=True, comm_mode="sum"))]


@pytest.mark.parametrize("name,B,family,over", FULL, ids=lambda v: str(v) if not isinstance(v, dict) else
                         "-".join("%s%s" % kv for kv in v.items()) or "p1")
def test_full_size_every_row_matches_float64(name, B, family, over):
    """81 920 rows.  max_steps 6 over 14 lock-steps: every slot starts three episodes; traffic junction has dead cars.
    Each step is fed from the trainer's records: the rollout's own value / log-probs and a direct step's h' against the
    float64 step."""
    tr = make_trainer(name, B, family, seed=5, id0=0, max_steps=6, **over)
    N, T = tr.args.nagents, 14
    R = B * N
    tr.rollout(T, 0)
    tr.collect_stat()                                    # raises on a device-side flag
    assert int(tr._buf["err"].item()) == 0
    b, net = tr._buf, tr.policy_net
    heads = tr.args.naction_heads
    tol = sum_tol(N) if over.get("comm_mode") == "sum" else ROW_TOL
    worst, nfresh, ndead = {}, 0, 0
    for t in range(T):
        inp = record_inputs(tr, t)
        ref, _ = ff_step_f64(net, inp["x"], B, inp["comm"], inp["alive"], inp["fresh"])
        out = outputs(R, heads)
        assert ff_direct_step(net, inp["x"], B, out, inp["comm"], inp["alive"], inp["fresh"]) == 0
        compare("%s %s step %d (direct)" % (name, family, t), {k: out[k] for k in ("h", "value", "logp")}, ref, worst, tol)
        compare("%s %s step %d (rollout)" % (name, family, t),
                dict(value=b["value"][t].reshape(R), logp=b["logp"][t].reshape(R, -1)), ref, worst, tol)
        nfresh += int(inp["fresh"].sum())
        ndead += int((inp["alive"] == 0).sum())
    assert nfresh > B and (ndead > 0 or not tr.is_tj)
    print("%s %s %s B=%d: %d rows x %d steps, worst |gpu - ref| / max(1, |ref|): %s" % (
        name, family, over, B, R, T, " ".join("%s %.2e" % kv for kv in worst.items())))


# ---------------------------------------------------------------------------------------------------- 2. fixtures

@pytest.mark.parametrize("name", ["var_mlp", "var_commnet_nonrec2"])
def test_forward_fixtures_of_the_reference(name):
    """The unmodified reference's forward (its state_dict, inputs, outputs) through policy_impl 'tc_ff'."""
    meta, z = load_golden(name)
    a, net = variant_net(meta, z, "tc_ff")
    assert net.policy_impl == "tc_ff"
    B, n = z["obs"].shape[0], a.nagents
    obs = torch.tensor(z["obs"], dtype=torch.float32, device="cuda")
    info = {}
    if meta["hard_attn"]:
        info["comm_action"] = torch.tensor(z["comm"], dtype=torch.uint8, device="cuda")
    if meta["use_alive"]:
        info["alive_mask"] = torch.tensor(z["alive"], dtype=torch.uint8, device="cuda")
    act, val = net(obs, info)
    torch.cuda.synchronize()
    net.check_errors()
    assert close(val.reshape(B, n).cpu().numpy(), z["value"])
    for k in range(len(meta["heads"])):
        assert close(act[k].cpu().numpy(), z["logp%d" % k]), k


def test_hid_size_32_fixture_is_refused():
    """var_commnet_nonrec_share is a hid_size 32 policy: outside the kernel, so 'tc_ff' refuses it (its forward stays on
    'simt', tests/test_gpu_variants.py)."""
    meta, z = load_golden("var_commnet_nonrec_share")
    assert meta["args"]["hid_size"] != 128
    with pytest.raises(NotImplementedError):
        variant_net(meta, z, "tc_ff")


@pytest.mark.parametrize("name", golden_names("gradff_"))
def test_gradient_fixtures_of_the_reference(name):
    """kernels_ff with the tc_ff forward: the pinned float64 oracle on 5 and 13 slots, and one slot against the
    reference's stored gradient arrays."""
    ff_pinned_oracle(name, 5, "tc_ff")
    ff_pinned_oracle(name, 13, "tc_ff")
    ff_gradient_arrays(name, "tc_ff")


# ---------------------------------------------------------------------------------------------------- 3. re-run

@pytest.mark.parametrize("name,family,over", [(PP, "ic3net", dict(comm_passes=3)),
                                              (TJ, "commnet", dict(comm_passes=2, share_weights=True, comm_mode="sum")),
                                              (PP, "mlp", {}), (PP, "commnet", dict(comm_passes=4))])
def test_rerun_equals_rollout_step(name, family, over):
    """ic3_policy_ff_states on the tc_ff weights: st_h[p] (p >= 1) equals the tc_ff ic3_policy_step cut to p passes bit
    for bit; st_h[0] is tanh(x); st_s[p] is the gated mean of st_h[p]."""
    from ic3net_b200 import _lib
    tr = make_trainer(name, 37, family, **over)
    tr.run_batch(0)
    net = tr.policy_net
    lib = _lib.load()
    B, N = tr.env.env.nenvs, tr.args.nagents
    R = B * N
    cfg, w = net.policy_cfg(B), net.packed()
    P = max(1, int(cfg.passes))
    inp = record_inputs(tr, tr._buf["T"] // 2)
    io = _lib.PolicyIO(x=inp["x"].data_ptr(), comm_action=_lib.ptr(inp["comm"]), alive=inp["alive"].data_ptr(),
                       fresh=inp["fresh"].data_ptr())
    st_h = torch.full((P + 1, R, 128), float("nan"), device="cuda")
    st_s = torch.full((P, R, 128), float("nan"), device="cuda")
    _lib.check(lib.ic3_policy_ff_states(C.byref(cfg), C.byref(w), C.byref(io), st_h.data_ptr(), st_s.data_ptr(),
                                        _lib.stream()))
    for p in range(1, P + 1):
        out = outputs(R, tr.args.naction_heads)
        assert ff_direct_step(net, inp["x"], B, out, inp["comm"], inp["alive"], inp["fresh"], passes=p) == 0
        assert torch.equal(st_h[p], out["h"]), p
    assert torch.allclose(st_h[0], torch.tanh(inp["x"]), rtol=0, atol=1e-6)
    g, den = gates_f64(B, N, inp["comm"], inp["alive"], inp["fresh"], bool(cfg.hard_attn), bool(cfg.comm_avg))
    if cfg.comm_mask_zero:
        g = torch.zeros_like(g)
    for p in range(P):
        hv = st_h[p].double().view(B, N, 128)
        want = gated_mean(hv, g, den)
        bound = 1e-6 * ((g * hv.abs()).sum(1, keepdim=True) + 1.0) / den      # fp32 rounding of the gated sum
        assert bool(((st_s[p].double().view(B, N, 128) - want).abs() <= bound).all()), p


# ---------------------------------------------------------------------------------------------------- 4. gradient

GRAD_FULL = [(n, fam, dict(comm_passes=p, share_weights=s)) for n in (PP, TJ)
             for fam, p, s in (("ic3net", 1, False), ("ic3net", 2, False), ("ic3net", 2, True), ("commnet", 4, False),
                               ("ic3net", 4, True))]


@pytest.mark.parametrize("name,family,over", GRAD_FULL + [(PP, "mlp", {})])
def test_full_size_gradient_matches_float64(name, family, over):
    ff_full_size(name, family, over, "tc_ff")


def test_gradient_is_bit_identical_run_to_run():
    ff_chunk_sizes_and_determinism("ic3net", dict(comm_passes=2), "tc_ff")
    ff_chunk_sizes_and_determinism("mlp", {}, "tc_ff")


@pytest.mark.parametrize("name,family,over", [(PP, "ic3net", dict(comm_passes=2)), (TJ, "commnet", dict(comm_passes=2))])
def test_halted_slots_contribute_nothing(name, family, over):
    ff_halted_slots_contribute_nothing(name, family, over, "tc_ff")


# ---------------------------------------------------------------------------------------------------- 5. row counts

def sweep_rows(case, ctas):
    return {"one-row": 1, "tile-1": TILE - 1, "tile+1": TILE + 1, "idle-CTAs": (ctas - 3) * TILE - 5,
            "grid": ctas * TILE, "grid+1": ctas * TILE + 1, "three-tiles": 2 * ctas * TILE + TILE + 3}[case]


@pytest.mark.parametrize("family,per_sm", [("mlp", 2), ("ic3net", 1)])
@pytest.mark.parametrize("case", ["one-row", "tile-1", "tile+1", "idle-CTAs", "grid", "grid+1", "three-tiles"])
def test_row_counts_and_rows_past_R(case, family, per_sm):
    """One agent per env, so R is any number, around the tile and the persistent grid (two CTAs per SM without
    communication, one with), two passes.  64 rows past R hold a NaN pattern and stay bit for bit; inputs stay."""
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    R, heads, extra = sweep_rows(case, per_sm * nsm), (5, 2), 64
    net = ff_net(1, heads, "tc_ff", family, passes=1 if family == "mlp" else 2, wseed=11)
    x, comm, alive, fresh = inputs(R, 1, seed=R)
    before = [t.clone() for t in (x, comm, alive, fresh)]
    out = outputs(R, heads, extra)
    pristine = {k: v.clone() for k, v in out.items()}
    assert ff_direct_step(net, x, R, out, comm, alive, fresh, draws=torch.zeros(R, 2, dtype=torch.int32, device="cuda")) == 0
    bits = lambda t: t.view(torch.int32) if t.dtype == torch.float32 else t
    for k, v in out.items():
        assert torch.equal(bits(v[R:]), bits(pristine[k][R:])), (case, k)
    for a, b in zip((x, comm, alive, fresh), before):
        assert torch.equal(a, b)
    ref, _ = ff_step_f64(net, x, R, comm, alive, fresh)
    compare("%s %s R=%d" % (family, case, R), {k: out[k][:R] for k in ("h", "value", "logp")}, ref)


@pytest.mark.parametrize("N", [1, 3, 10, 20, 22, 32])
@pytest.mark.parametrize("family,passes,mode", [("ic3net", 2, "avg"), ("commnet", 3, "sum"), ("mlp", 1, "avg")])
def test_agents_per_env(N, family, passes, mode):
    """floor(64 / N) envs per tile with 64 mod N padding rows; dead agents, fresh slots, silent agents; 257 envs leave a
    ragged last tile.  Rows past R stay untouched."""
    B, heads, extra = 257, (5,), 64
    R = B * N
    net = ff_net(N, heads, "tc_ff", family, passes=passes, mode=mode, wseed=N)
    x, comm, alive, fresh = inputs(B, N, seed=N)
    out = outputs(R, heads, extra)
    assert ff_direct_step(net, x, B, out, comm, alive, fresh) == 0
    assert torch.isnan(out["h"][R:]).all() and bool((out["action"][R:] == -7).all())
    ref, _ = ff_step_f64(net, x, B, comm, alive, fresh)
    worst = {}
    compare("%s N=%d" % (family, N), {k: out[k][:R] for k in ("h", "value", "logp")}, ref, worst,
            sum_tol(N) if mode == "sum" else ROW_TOL)
    print("%s %d passes %s N=%d: %s" % (family, passes, mode, N, " ".join("%s %.2e" % kv for kv in worst.items())))


# ---------------------------------------------------------------------------------------------------- 6. sampling

@pytest.mark.parametrize("family", ["mlp", "ic3net"])
@pytest.mark.parametrize("heads", [(5,), (5, 2), (9, 8), (16, 15)], ids=lambda h: "x".join(map(str, h)))
def test_sampling_with_explicit_draws(heads, family):
    """Explicit draws: u24 = 0, 2^24 - 1, draws on the float64 CDF edges and random ones.  Actions are in range, equal the
    float64 inverse CDF away from the edges, and equal the SIMT path's wherever both paths' log-probs put the draw on
    the same side of every CDF edge."""
    N, B = 7, 300
    R = B * N
    tc, simt = twin_nets(N, heads, family, wseed=sum(heads))
    x, comm, alive, fresh = inputs(B, N, seed=sum(heads))
    rs = np.random.RandomState(1)
    u24 = rs.randint(0, 1 << 24, size=(R, len(heads))).astype(np.int64)
    rows = np.arange(R)
    u24[rows % 8 == 0] = 0
    u24[rows % 8 == 1] = (1 << 24) - 1
    ref, _ = ff_step_f64(tc, x, B, comm, alive, fresh)
    off = 0
    for k, na in enumerate(heads):
        cdf = np.cumsum(np.exp(ref["logp"][:, off:off + na].cpu().numpy()), -1)
        edge = cdf[rows, rs.randint(0, max(na - 1, 1), R)] * (1 << 24)
        on = (rows % 8 == 2) | (rows % 8 == 3)
        u24[on, k] = np.clip(np.where(rows[on] % 8 == 2, np.floor(edge[on]), np.ceil(edge[on])), 0, (1 << 24) - 1)
        off += na
    draws = torch.as_tensor(u24.astype(np.int32), device="cuda").contiguous()
    o_tc, o_simt = outputs(R, heads), outputs(R, heads)
    assert ff_direct_step(tc, x, B, o_tc, comm, alive, fresh, draws=draws) == 0
    assert ff_direct_step(simt, x, B, o_simt, comm, alive, fresh, draws=draws) == 0
    compare("heads %s" % (heads,), {k: o_tc[k] for k in ("h", "value", "logp")}, ref)
    a_tc, a_simt = o_tc["action"].cpu().numpy(), o_simt["action"].cpu().numpy()
    off = 0
    for k, na in enumerate(heads):
        assert a_tc[:, k].min() >= 0 and a_tc[:, k].max() < na
        want, margin = inverse_cdf(ref["logp"][:, off:off + na], u24[:, k])
        assert not np.any((margin > MARGIN) & (want != a_tc[:, k])), (heads, k)
        w_tc, m_tc = inverse_cdf(o_tc["logp"][:, off:off + na], u24[:, k])
        w_simt, m_simt = inverse_cdf(o_simt["logp"][:, off:off + na], u24[:, k])
        same = (w_tc == w_simt) & (m_tc > MARGIN) & (m_simt > MARGIN)
        assert same.mean() > 0.7 and np.array_equal(a_tc[same, k], a_simt[same, k]), (heads, k)
        off += na


# ---------------------------------------------------------------------------------------------------- 7. fp16 range

@pytest.mark.parametrize("which", ["f", "c"])
def test_weight_limit_of_the_fp16_split(which):
    """|w| * 256 must stay below 65504: an entry of 255 in F_1 (or C_1) raises no flag and meets the bar, one of 256 is
    refused with the fp16-range flag (0x200), not computed with a saturated weight."""
    N, B, heads = 10, 40, (5,)
    x, comm, alive, fresh = inputs(B, N, seed=2, scale=1e-3)
    for entry, ok in ((255.0, True), (256.0, False)):
        net = ff_net(N, heads, "tc_ff", "commnet", passes=2, wseed=13)
        with torch.no_grad():
            (net.f_modules[1] if which == "f" else net.C_modules[1]).weight[3, 7] = entry
        out = outputs(B * N, heads)
        flags = ff_direct_step(net, x, B, out, comm, alive, fresh)
        if ok:
            assert flags == 0
            ref, _ = ff_step_f64(net, x, B, comm, alive, fresh)
            compare("|w| 255", {k: out[k] for k in ("h", "value", "logp")}, ref)
        else:
            assert flags == 0x200


def test_largest_sum_mode_communication_stays_in_range():
    """comm_mode sum, 32 agents all alive and talking, every h near 1: S reaches 31 (16 S = 496 in fp16) and the step
    meets the bar with no flag."""
    N, B, heads = 32, 50, (5,)
    net = ff_net(N, heads, "tc_ff", "commnet", passes=2, mode="sum", wseed=4)
    with torch.no_grad():
        for m in net.C_modules:
            m.weight.mul_(0.01)
    x = torch.full((B * N, 128), 6.0, device="cuda")
    out = outputs(B * N, heads)
    assert ff_direct_step(net, x, B, out) == 0
    assert float(torch.tanh(x.double()).min()) * (N - 1) > 30.9
    ref, _ = ff_step_f64(net, x, B)
    compare("sum S = 31", {k: out[k] for k in ("h", "value", "logp")}, ref, tol=sum_tol(N))


# ---------------------------------------------------------------------------------------------------- 8. graph

@pytest.mark.parametrize("obs_mode", ["index", "dense"])
def test_graph_rollout_equals_eager(obs_mode):
    recs = []
    for use_graph in (False, True):
        tr = make_trainer(PP, 96, "ic3net", comm_passes=2, seed=3, id0=1, max_steps=7, obs_mode=obs_mode,
                          use_graph=use_graph)
        tr.rollout(16, 0)
        tr.collect_stat()
        b = tr._buf
        recs.append({k: b[k].clone() for k in ("value", "logp", "action", "reward")})
    for k in recs[0]:
        assert torch.equal(recs[0][k], recs[1][k]), (obs_mode, k)


@pytest.mark.parametrize("family", ["mlp", "ic3net"])
def test_autograd_gradient_with_tc_ff_rollout(family):
    """grad_impl 'autograd' recomputes the step in torch from the rollout's records; with the tc_ff rollout it agrees
    with kernels_ff on the same rollout."""
    ka = make_trainer(PP, 48, family, comm_passes=2 if family != "mlp" else 1)
    au = make_trainer(PP, 48, family, grad_impl="autograd", comm_passes=2 if family != "mlp" else 1)
    gk, sk = rollout_and_grad(ka)
    ga, sa = rollout_and_grad(au)
    assert_close(gk, sk, ga, sa)
    assert int(ka._buf["err"].item()) == 0 and int(au._buf["err"].item()) == 0


# ---------------------------------------------------------------------------------------------------- 9. refusals

def test_refusals_and_default():
    from ic3net_b200 import models
    from ic3net_b200.comm import CommNetMLP
    base = dict(nagents=3, hid_size=128, comm_passes=1, recurrent=True, rnn_type="LSTM", continuous=False,
                naction_heads=[5], comm_mask_zero=False, comm_mode="avg", hard_attn=False, comm_init="uniform",
                share_weights=False, seed=0, env_id0=0, commnet=True, policy_impl="tc_ff")
    with pytest.raises(NotImplementedError, match="'tc'"):                  # recurrent CommNet / IC3Net (LSTM)
        CommNetMLP(argparse.Namespace(**base), 29)
    with pytest.raises(NotImplementedError, match="tc_tanh"):               # IC / IRIC (tanh RNN)
        models.RNN(argparse.Namespace(**dict(base, rnn_type="MLP")), 29)
    with pytest.raises(NotImplementedError):                                # models.RNN with the LSTM cell
        models.RNN(argparse.Namespace(**base), 29)
    with pytest.raises(NotImplementedError):                                # hid_size 64
        ff_net(3, (5,), "tc_ff", "ic3net", H=64)
    net = ff_net(3, (5,), None, "ic3net")
    assert net.policy_impl == "simt" and net.workspace(4) == (None, None)
    assert ff_net(3, (5,), None, "mlp").policy_impl == "simt"
    for impl in ("tc", "tc_tanh"):                                          # the existing refusals stay
        with pytest.raises(NotImplementedError):
            ff_net(3, (5,), impl, "commnet")


# ---------------------------------------------------------------------------------------------------- 10. CLI

def test_command_line(capsys):
    from ic3net_b200 import main as cli
    rc = cli.main(["--env_name", "predator_prey", "--nagents", "3", "--dim", "5", "--max_steps", "20", "--hid_size", "128",
                   "--commnet", "--comm_passes", "2", "--policy_impl", "tc_ff", "--grad_impl", "kernels_ff", "--nenvs",
                   "64", "--num_epochs", "1", "--epoch_size", "1", "--batch_size", "40"])
    out = capsys.readouterr().out
    assert rc == 0 and "Epoch" in out, out[-2000:]
