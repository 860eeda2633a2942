"""GPU tests of the tensor-core policy step (csrc/policy_tc.cu: prep_kernel -> lstm_tc_kernel -> heads_finish_kernel /
heads_kernel<P>, weights from pack_tc_kernel) on EVERY row against the batched float64 step of tests/policy_ref.py.

Covered: the full batch sizes of predator-prey hard (8192 envs) and traffic-junction hard (4096 envs), 81 920 rows per
step, every step of a rollout with episode resets, from the trainer's own records; row counts around the thresholds of
the persistent LSTM kernel (derived from the card's SM count: one or several work items per CTA, padding tiles, ragged
last tiles, an empty second warpgroup) on the tensor-core and the fp32 SIMT path; comm_passes > 1, share_weights and the
other comm variants beyond one tile; every branch of the heads (fused epilogue, heads_kernel<16>, heads_kernel<32>) with
explicit draws; the rows past R; and both sides of the fp16 operand-split limits.

Bar: |gpu - ref| <= 1e-5 * max(1, |ref|) on h', c', value and log-probs (DESIGN.md section 2).  A failure names the worst
element's row, 128-row tile, warpgroup, column half, work item and CTA of lstm_tc_kernel."""
import numpy as np
import pytest
import torch

from gpu_harness import (MARGIN, TC_TILE, TC_TILE_PAD, compare_rows, lstm_direct_step, lstm_outputs, make_lstm_net,
                         params_f64, ref_dict, rows_trainer, sms, step_f64, synthetic, tc_geometry, tc_where,
                         trainer_rows)
from helpers import load_golden
from policy_ref import inverse_cdf

pytestmark = pytest.mark.gpu


def compare(label, got, ref, worst=None):
    """Every row of got against ref at the bar, a failure named in lstm_tc_kernel's work decomposition."""
    return compare_rows(label, got, ref, worst, where=tc_where(ref["value"].shape[0]))



# ---------------------------------------------------------------------------------------------------- policies

def reference(net, a, obs, h, c, comm, alive):
    B, N, O = obs.shape
    P = params_f64(net.state_dict(), a.comm_passes, device="cuda")
    return ref_dict(*step_f64(P, obs.reshape(B * N, O).double(), h, c, comm if a.hard_attn else None, alive, None,
                              nagents=N, passes=a.comm_passes, hard_attn=a.hard_attn, comm_mode=a.comm_mode,
                              comm_mask_zero=a.comm_mask_zero))


def forward(net, a, obs, h, c, comm, alive):
    info = {"alive_mask": alive}
    if a.hard_attn:
        info["comm_action"] = comm
    act, val, (h2, c2) = net([obs, (h, c)], info)
    torch.cuda.synchronize()
    if net.policy_impl == "tc":
        net.check_errors()
    return dict(h=h2, c=c2, value=val, logp=torch.cat(act, -1))


# ---------------------------------------------------------------------------------------------------- a. full size

@pytest.mark.parametrize("name,B", [("grad_pp_hard_ic3net_h128", 8192), ("grad_tj_hard_ic3net_h128", 4096)])
def test_full_size_every_row_matches_float64(name, B):
    """81 920 rows: 640 tiles, 1280 work items, nine or ten items per CTA.  max_steps 6 over 14 lock-steps: every slot
    starts three episodes, so the fresh branches of the operand preparation and of the epilogue run at full size."""
    tr = rows_trainer(name, B, max_steps=6)
    assert tr.grad_kernels
    trainer_rows(tr, 14, "%s B=%d" % (name, B), sensitivity=True)


# ---------------------------------------------------------------------------------------------------- b. row sweep

def sweep_batch(case, N, nsm):
    """Env slots B (N agents each) giving the row / tile / work-item count the case is about."""
    def with_tiles(nt):                                  # R just past nt - 1 tiles: the last tile holds 1..N rows
        return ((nt - 1) * TC_TILE) // N + 1
    if case == "R<64":
        return 63 // N
    if case == "64<R<128":
        return 127 // N
    if case == "R=128k+1":
        return next(b for b in range(1, 1 << 16) if (b * N) % TC_TILE == 1 and b * N > 2 * TC_TILE)
    if case == "no-padding-tiles":
        return 1024                                      # R = 1024 N: 8 N tiles
    if case == "7-padding-tiles":
        return with_tiles(17)
    if case == "items<SMs":
        return with_tiles((nsm - 1) // 16 * 8 - 3)       # padded to (nsm - 1) // 16 * 8 tiles
    if case == "items>SMs":
        return with_tiles((nsm // 16 + 1) * 8)
    if case == "items>=3SMs":
        ntp = -(-(3 * nsm + 1) // 16) * 8
        if (2 * ntp) % nsm == 0:
            ntp += 8
        return with_tiles(ntp)
    raise KeyError(case)


def sweep_checks(case, B, N, nsm):
    R = B * N
    nt, ntp, items, grid = tc_geometry(R)
    ok = {"R<64": R < 64, "64<R<128": 64 < R < 128, "R=128k+1": R % TC_TILE == 1 and nt >= 3,
          "no-padding-tiles": R % TC_TILE == 0 and nt % TC_TILE_PAD == 0,
          "7-padding-tiles": nt % TC_TILE_PAD == 1,
          "items<SMs": items < nsm, "items>SMs": nsm < items < 2 * nsm,
          "items>=3SMs": items >= 3 * nsm and items % nsm != 0}[case]
    assert ok, (case, B, N, R, nt, ntp, items, nsm)
    return "%s N=%d B=%d R=%d tiles=%d (padded %d) items=%d CTAs=%d SMs=%d" % (case, N, B, R, nt, ntp, items, grid, nsm)


SWEEP = [("R<64", 7), ("R<64", 20), ("R<64", 32), ("64<R<128", 3), ("64<R<128", 10), ("64<R<128", 32),
         ("R=128k+1", 1), ("R=128k+1", 3), ("R=128k+1", 7), ("no-padding-tiles", 10), ("no-padding-tiles", 32),
         ("7-padding-tiles", 2), ("7-padding-tiles", 7), ("items<SMs", 3), ("items<SMs", 20), ("items>SMs", 7),
         ("items>SMs", 10), ("items>=3SMs", 1), ("items>=3SMs", 10), ("items>=3SMs", 32)]


@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("case,N", SWEEP)
def test_row_and_work_item_sweep(case, N, impl):
    """CommNetMLP.forward at row counts chosen from the SM count (an empty second warpgroup, a partial tile, one row in
    the last tile, no padding tiles, seven padding tiles, one item per CTA with idle CTAs, CTAs with two items, the ring
    phase carried over three or more items with uneven CTAs); every row against float64.  The SIMT kernel runs the same
    batches (64-row whole-env tiles)."""
    nsm = sms()
    B = sweep_batch(case, N, nsm)
    label = sweep_checks(case, B, N, nsm) + " " + impl
    O = 61
    net, a = make_lstm_net(N, O, (5, 2), wseed=N, impl=impl)
    inputs = synthetic(B, N, O, seed=1000 * N + len(case))
    errs = compare(label, forward(net, a, *inputs), reference(net, a, *inputs))
    print(label, " ".join("%s %.2e" % kv for kv in errs.items()))


# ---------------------------------------------------------------------------------------------------- c. variants

VARIANTS = [dict(passes=2), dict(passes=3), dict(passes=3, share=True, hard_attn=False), dict(passes=2, share=True),
            dict(hard_attn=False), dict(comm_mode="sum"), dict(comm_mask_zero=True)]


@pytest.mark.parametrize("kw", VARIANTS, ids=["-".join("%s=%s" % i for i in v.items()) for v in VARIANTS])
def test_variants_beyond_one_tile(kw):
    """Tensor-core path at the 'items >= 3 x SMs' size: comm_passes 2 and 3 (the odd count reuses carry buffer 0),
    share_weights, soft attention, comm_mode sum and comm_mask_zero, every row against float64."""
    N, O = 10, 61
    nsm = sms()
    B = sweep_batch("items>=3SMs", N, nsm)
    label = sweep_checks("items>=3SMs", B, N, nsm) + " " + str(kw)
    net, a = make_lstm_net(N, O, (5, 2), wseed=7, **kw)
    assert net.policy_impl == "tc"
    inputs = synthetic(B, N, O, seed=77)
    errs = compare(label, forward(net, a, *inputs), reference(net, a, *inputs))
    print(label, " ".join("%s %.2e" % kv for kv in errs.items()))


def test_enemy_comm_rollout_beyond_one_tile():
    """--enemy_comm (the prey is agent row N - 1 of every env) in a trainer rollout at the 'items >= 3 x SMs' size."""
    name = "grad_pp_enemy_ic3net_h128"
    N = load_golden(name)[0]["args"]["nagents"]
    nsm = sms()
    B = sweep_batch("items>=3SMs", N, nsm)
    label = sweep_checks("items>=3SMs", B, N, nsm) + " enemy_comm"
    tr = rows_trainer(name, B, seed=9, id0=4, max_steps=5)
    trainer_rows(tr, 12, label)


def test_two_pass_rollout_with_resets():
    """comm_passes = 2 in a trainer rollout with episode resets: the recorded values / log-probs and the state entering
    every next step against float64 replayed over the trainer's own (h, c) checkpoints."""
    name = "grad_pp_hard_ic3net_h128"
    tr = rows_trainer(name, 1024, seed=21, id0=2, comm_passes=2, max_steps=5, grad_impl="autograd")
    assert tr.policy_net.policy_impl == "tc" and tr.policy_net.is_variant and not tr.grad_kernels
    trainer_rows(tr, 12, "pp hard comm_passes=2 B=1024")


# ---------------------------------------------------------------------------------------------------- d. heads

HEADS = [(5, 2), (2, 2, 2, 1), (9, 2), (5, 5, 5), (3, 4, 2, 5), (9, 8), (16, 15), (8, 8, 8, 7)]


@pytest.mark.parametrize("heads", HEADS, ids=["x".join(map(str, h)) for h in HEADS])
def test_heads_with_explicit_draws(heads):
    """1 + sum(heads) = 8 (fused into the LSTM epilogue, heads_finish_kernel), 9..16 (heads_kernel<16>), 17..32
    (heads_kernel<32>), four heads.  Values / log-probs against float64; actions against the float64 inverse CDF away
    from the CDF edges, and in range everywhere: u24 = 0, u24 = 2^24 - 1 and draws placed on the float64 CDF edges."""
    N, O, B = 7, 61, 300
    R = B * N
    nout = 1 + sum(heads)
    net, a = make_lstm_net(N, O, heads, wseed=sum(heads))
    inputs = synthetic(B, N, O, seed=nout)
    ref = reference(net, a, *inputs)
    rs = np.random.RandomState(nout)
    u24 = rs.randint(0, 1 << 24, size=(R, len(heads))).astype(np.int64)
    rows = np.arange(R)
    u24[rows % 8 == 0] = 0
    u24[rows % 8 == 1] = (1 << 24) - 1
    off = 0
    for k, na in enumerate(heads):
        cdf = np.cumsum(np.exp(ref["logp"][:, off:off + na].cpu().numpy()), -1)
        edge = cdf[rows, rs.randint(0, max(na - 1, 1), R)] * (1 << 24)
        on = (rows % 8 == 2) | (rows % 8 == 3)
        u24[on, k] = np.clip(np.where(rows[on] % 8 == 2, np.floor(edge[on]), np.ceil(edge[on])), 0, (1 << 24) - 1)
        off += na
    draws = torch.as_tensor(u24.astype(np.int32), device="cuda").contiguous()
    out = lstm_outputs(R, heads)
    assert lstm_direct_step(net, *inputs, out, draws=draws) == 0
    label = "heads %s (%d outputs)" % (heads, nout)
    errs = compare(label, out, ref)
    act = out["action"].cpu().numpy()
    off, safe_total = 0, 0
    for k, na in enumerate(heads):
        assert act[:, k].min() >= 0 and act[:, k].max() < na, (label, k)
        want, margin = inverse_cdf(ref["logp"][:, off:off + na], u24[:, k])
        safe = margin > MARGIN
        bad = np.nonzero(safe & (want != act[:, k]))[0]
        assert bad.size == 0, (label, k, bad[:10], u24[bad[:10], k])
        safe_total += int(safe.sum())
        off += na
    assert safe_total > R * len(heads) // 2
    print(label, " ".join("%s %.2e" % kv for kv in errs.items()))


# ---------------------------------------------------------------------------------------------------- e. rows past R

@pytest.mark.parametrize("heads,passes", [((5, 2), 1), ((9, 8), 1), ((5, 2), 2)])
@pytest.mark.parametrize("case", ["R=128k+1", "7-padding-tiles"])
def test_writes_stay_inside_the_rows(case, heads, passes):
    """Outputs with 64 extra rows past R, filled with a NaN bit pattern: the ragged last tile and the padding tiles must
    leave them bit for bit unchanged, and the step must not write its inputs."""
    N, O, extra = 7, 61, 64
    nsm = sms()
    B = sweep_batch(case, N, nsm)
    label = sweep_checks(case, B, N, nsm) + " heads %s passes %d" % (heads, passes)
    R = B * N
    net, a = make_lstm_net(N, O, heads, wseed=11, passes=passes)
    obs, h, c, comm, alive = synthetic(B, N, O, seed=5)
    before = [t.clone() for t in (obs, h, c, comm, alive)]
    out = lstm_outputs(R, heads, extra)
    pristine = {k: v.clone() for k, v in out.items()}
    assert lstm_direct_step(net, obs, h, c, comm, alive, out,
                       draws=torch.zeros(R, len(heads), dtype=torch.int32, device="cuda")) == 0
    for k, v in out.items():
        bits = lambda t: t.view(torch.int32) if t.dtype == torch.float32 else t
        assert torch.equal(bits(v[R:]), bits(pristine[k][R:])), (label, k)
    for x, y in zip((obs, h, c, comm, alive), before):
        assert torch.equal(x, y), label
    compare(label, {k: v[:R] for k, v in out.items()}, reference(net, a, obs, h, c, comm, alive))


# ---------------------------------------------------------------------------------------------------- f. fp16 limits

def limit_case(enc_bias=None, c_entry=None, small=False):
    """A 10-agent policy at the 'items > SMs' size with one parameter pushed to an fp16 split limit.  Returns
    (device flag word, got, ref)."""
    N, O = 10, 61
    B = sweep_batch("items>SMs", N, sms())
    net, a = make_lstm_net(N, O, (5, 2), wseed=13)
    obs, h, c, comm, alive = synthetic(B, N, O, seed=13, h_scale=1e-4 if small else 1.0, c_scale=1e-4 if small else 3.0)
    with torch.no_grad():
        if enc_bias is not None:
            # unit 5 of x sits at enc_bias (its observation weights scaled down so that it stays there); the W_ih column
            # it meets is scaled down too, so that the gates stay unsaturated and the check measures the operand split
            # rather than the fp32 rounding of x itself (half an ulp is 1.2e-4 there)
            net.encoder.bias[5] = enc_bias
            net.encoder.weight[5] *= 1e-3
            net.f_module.weight_ih[:, 5] *= 1e-3
        if c_entry is not None:
            # (W_ih . C)[0][0] = 1 * c_entry is the largest folded weight; every other one stays far below 255
            net.C_modules[0].weight.zero_()
            net.C_modules[0].weight[0, 0] = c_entry
            net.f_module.weight_ih[0, 0] = 1.0
        if small:
            net.encoder.weight.mul_(1e-4)
            net.encoder.bias.mul_(1e-4)
    R = B * N
    out = lstm_outputs(R, (5, 2))
    flags = lstm_direct_step(net, obs, h, c, comm, alive, out, draws=torch.zeros(R, 2, dtype=torch.int32, device="cuda"))
    return flags, out, reference(net, a, obs, h, c, comm, alive), net, obs


def test_activation_limit_of_the_fp16_split():
    """|x| * 16 must stay below 65504: max |x| = 4090 raises no flag and meets the bar, 4100 raises IC3_ERR_FP16_RANGE."""
    flags, out, ref, net, obs = limit_case(enc_bias=4090.0)
    x = obs.reshape(-1, obs.shape[-1]).double() @ net.encoder.weight.detach().double().t() + \
        net.encoder.bias.detach().double()
    assert 4089 < float(x.abs().max()) < 4091
    assert flags == 0, hex(flags)
    compare("max |x| %.1f" % float(x.abs().max()), out, ref)
    flags, _, _, _, _ = limit_case(enc_bias=4100.0)
    assert flags == 0x200, hex(flags)


def test_folded_weight_limit_of_the_fp16_split():
    """|W_ih . C| * 256 must stay below 65504: an entry of 255 raises no flag, one of 256 does."""
    flags, _, _, _, _ = limit_case(c_entry=255.0)
    assert flags == 0, hex(flags)
    flags, _, _, _, _ = limit_case(c_entry=256.0)
    assert flags == 0x200, hex(flags)


def test_tiny_activations_with_subnormal_low_halves():
    """x, h and c around 1e-4: the low fp16 half of each operand (2^-11 of its 16-fold value) is subnormal."""
    flags, out, ref, net, obs = limit_case(small=True)
    assert flags == 0, hex(flags)
    x = obs.reshape(-1, obs.shape[-1]).double() @ net.encoder.weight.detach().double().t() + \
        net.encoder.bias.detach().double()
    assert float(x.abs().max()) < 1e-3
    compare("activations ~1e-4", out, ref)
