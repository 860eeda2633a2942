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
import argparse
import ctypes as C

import numpy as np
import pytest
import torch

from bptt_ref import tj_record_obs
from helpers import finish_args, load_golden, ns
from oracle import philox
from oracle.gen_golden import make_weights
from policy_ref import inverse_cdf, params_f64, philox_u24, step_f64

pytestmark = pytest.mark.gpu

TOL = 1e-5
MARGIN = 1e-5               # draws closer than this to a CDF edge may flip between fp32 and float64
TILE, TILE_PAD = 128, 8     # rows per tile; tiles are padded to a multiple of 8 (csrc/policy_tc.cu)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def geometry(R):
    """(tiles, padded tiles, work items, CTAs) of lstm_tc_kernel for R rows: one item per (tile, 64-unit column half),
    a persistent grid of min(items, SMs) CTAs (one resident CTA per SM)."""
    nt = -(-R // TILE)
    ntp = -(-nt // TILE_PAD) * TILE_PAD
    return nt, ntp, 2 * ntp, min(2 * ntp, sms())


def rel_err(got, ref):
    got, ref = got.to(torch.float64), ref.to(torch.float64)
    return ((got - ref).abs() / ref.abs().clamp_min(1.0)).reshape(ref.shape[0], -1)


def where(err, R, unit_cols):
    """Where the worst element of err [R, W] sits in the kernel's work decomposition."""
    r, col = divmod(int(err.argmax()), err.shape[1])
    _, _, items, grid = geometry(R)
    tile, wg = r // TILE, (r % TILE) // 64
    if unit_cols:            # h', c': hidden unit `col` belongs to the column half col // 64
        half = col // 64
        item = 2 * tile + half
        return "row %d col %d: tile %d, warpgroup %d, column half %d, item %d, CTA %d (of %d, %d items)" % (
            r, col, tile, wg, half, item, item % grid, grid, items)
    return "row %d col %d: tile %d, warpgroup %d, items %d/%d, CTAs %d/%d (of %d)" % (
        r, col, tile, wg, 2 * tile, 2 * tile + 1, (2 * tile) % grid, (2 * tile + 1) % grid, grid)


def compare(label, got, ref, worst=None):
    """got / ref: dicts of h, c [R, H], value [R], logp [R, A] (h, c may be absent from got).  Asserts the bar;
    returns {output: max error}."""
    errs, msgs = {}, []
    R = ref["value"].shape[0]
    for k in ("h", "c", "value", "logp"):
        if k not in got:
            continue
        e = rel_err(got[k].reshape(R, -1), ref[k].reshape(R, -1))
        errs[k] = float(e.max())
        if worst is not None:
            worst[k] = max(worst.get(k, 0.0), errs[k])
        if not errs[k] <= TOL:
            nbad = int((e > TOL).any(1).sum())
            msgs.append("%s: %s max %.3e at %s; %d rows over the bar" % (label, k, errs[k], where(e, R, k in "hc"),
                                                                      nbad))
    assert not msgs, "\n".join(msgs)
    return errs


def ref_dict(h, c, value, logps):
    return dict(h=h, c=c, value=value, logp=torch.cat(logps, -1))


# ---------------------------------------------------------------------------------------------------- policies

def policy_args(N, heads, hard_attn=True, comm_mode="avg", comm_mask_zero=False, passes=1, share=False, impl="tc"):
    return argparse.Namespace(nagents=N, hid_size=128, comm_passes=passes, recurrent=True, rnn_type="LSTM",
                              continuous=False, naction_heads=list(heads), comm_mask_zero=comm_mask_zero,
                              comm_mode=comm_mode, hard_attn=hard_attn, comm_init="uniform", share_weights=share,
                              seed=0, env_id0=0, commnet=True, policy_impl=impl)


def make_net(N, O, heads, wseed=3, **kw):
    """CommNetMLP with the weights of make_weights (one comm pass) or, with comm_passes > 1, its own seeded init."""
    from ic3net_b200.comm import CommNetMLP
    a = policy_args(N, heads, **kw)
    torch.manual_seed(wseed)
    net = CommNetMLP(a, O)
    if a.comm_passes == 1:
        sd = make_weights(wseed, O, 128, heads)
        net.load_state_dict({k: torch.from_numpy(v).float() for k, v in sd.items()})
    return net, a


def synthetic(B, N, O, seed, h_scale=1.0, c_scale=3.0):
    """Sparse integer observations, h in [-1, 1], c in [-3, 3], random comm / alive masks; env b % 4 == 0 has nobody
    alive, b % 4 == 1 exactly one agent, b % 4 == 2 everybody."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    dev = "cuda"
    obs = ((torch.rand(B, N, O, generator=g, device=dev) < 0.1) *
           torch.randint(1, 4, (B, N, O), generator=g, device=dev)).float()
    h = (torch.rand(B * N, 128, generator=g, device=dev) * 2 - 1) * h_scale
    c = (torch.rand(B * N, 128, generator=g, device=dev) * 2 - 1) * c_scale
    comm = torch.randint(0, 2, (B, N), generator=g, device=dev, dtype=torch.uint8)
    alive = torch.randint(0, 2, (B, N), generator=g, device=dev, dtype=torch.uint8)
    kind = torch.arange(B, device=dev) % 4
    alive[kind == 0] = 0
    one = torch.zeros(N, dtype=torch.uint8, device=dev)
    one[N // 2] = 1
    alive[kind == 1] = one
    alive[kind == 2] = 1
    return obs, h, c, comm, alive


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

def make_trainer(name, B, seed=5, id0=0, **over):
    """Trainer (tensor-core policy, index observations, records for the gradient) on fixture ``name``'s arguments and
    weights.  With the BPTT kernels the records hold every step's (h, c) (rec_h / rec_c); otherwise grad_window = 1
    checkpoints (h, c) before every step (ck_h / ck_c)."""
    from ic3net_b200 import data
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    meta, _ = load_golden(name)
    args = ns(meta["args"], nenvs=B, seed=seed, env_id0=id0, obs_mode="index", use_graph=False, policy_impl="tc",
              record_for_grad=True, grad_window=1, **over)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    torch.manual_seed(meta["weights_seed"])
    net = CommNetMLP(args, args.num_inputs)
    if int(args.comm_passes) == 1:
        sd = make_weights(meta["weights_seed"], args.num_inputs, args.hid_size, args.naction_heads, args.comm_init)
        net.load_state_dict({k: torch.from_numpy(v).float() for k, v in sd.items()})
    return Trainer(args, net, env)


def trainer_rows(tr, T, label, sensitivity=False):
    """One rollout of T lock-steps, then every row of every step against step_f64 from the recorded state entering the
    step, the recorded observation state and masks.  Recorded actions are recomputed from the reference's log-probs
    with the trainer's own Philox draws.  Returns {output: worst error}."""
    e, args = tr.env.env, tr.args
    B, N = e.nenvs, args.nagents
    R = B * N
    tick0 = e.tick.clone().to(torch.int64).cpu().numpy()
    tr.rollout(T, 0)
    tr.collect_stat()                                    # raises on a device-side flag
    b = tr._buf
    gk = tr.grad_kernels
    hs, cs = (b["rec_h"], b["rec_c"]) if gk else (b["ck_h"], b["ck_c"])
    passes = int(args.comm_passes)
    P = params_f64(tr.policy_net.state_dict(), passes, device="cuda")
    kw = dict(nagents=N, passes=passes, hard_attn=bool(args.hard_attn) and bool(args.commnet),
              comm_mode=getattr(args, "comm_mode", "avg"), comm_mask_zero=bool(args.comm_mask_zero))
    seed, id0 = int(e.cfg.seed), int(e.cfg.env_id0)
    heads = list(args.naction_heads)

    def obs(t):
        if tr.is_tj:
            return tj_record_obs(tr, t, 0, B).reshape(R, -1).double()
        idx, val = tr._pp_sparse_obs(b["s_loc"][t])
        return idx, val.double()

    worst, flips, draws, nfresh = {}, 0, 0, 0
    for t in range(T):
        ref = ref_dict(*step_f64(P, obs(t), hs[t], cs[t], b["s_comm"][t], b["s_alive"][t], b["s_fresh"][t], **kw))
        nfresh += int(b["s_fresh"][t].sum())
        got = dict(value=b["value"][t], logp=b["logp"][t].reshape(R, -1))
        if gk or t + 1 < T:                              # checkpoints (ck_h) hold the state entering steps 0 .. T-1
            got.update(h=hs[t + 1], c=cs[t + 1])
        compare("%s step %d" % (label, t), got, ref, worst)
        # actions: the draws of (seed, env_id0 + b, tick, agent), inverse CDF on the float64 log-probs
        u24 = philox_u24(seed, id0 + np.arange(B)[:, None], (tick0 + t)[:, None], philox.STREAM_ACTION,
                         np.arange(N)[None, :]).reshape(R, 4)
        act = b["action"][t].reshape(R, -1).cpu().numpy()
        off = 0
        for k, na in enumerate(heads):
            want, margin = inverse_cdf(ref["logp"][:, off:off + na], u24[:, k])
            safe = margin > MARGIN
            bad = np.nonzero(safe & (want != act[:, k]))[0]
            assert bad.size == 0, "%s step %d head %d: action differs at rows %s" % (label, t, k, bad[:10])
            flips += int((want != act[:, k]).sum())
            draws += R
            off += na
    assert flips <= 1e-3 * draws, (flips, draws)
    assert nfresh > B, "every slot must start an episode again inside the rollout"
    print("%s: %d rows x %d steps, worst |gpu - ref| / max(1, |ref|): %s; action flips at CDF edges %d of %d" % (
        label, R, T, " ".join("%s %.2e" % kv for kv in worst.items()), flips, draws))
    if sensitivity:
        show_sensitivity(tr, P, obs, hs, cs, kw, label)
    return worst


def show_sensitivity(tr, P, obs, hs, cs, kw, label):
    """The comparison notices a one-env mix-up and a dropped episode reset: both modified references break the bar."""
    b, N = tr._buf, kw["nagents"]
    fr = b["s_fresh"]
    got = lambda t: dict(h=hs[t + 1], c=cs[t + 1], value=b["value"][t], logp=b["logp"][t].reshape(hs[t].shape[0], -1))
    # in the middle of an episode, env's h taken from its neighbour env + 1 (the pair whose states differ most: traffic-
    # junction envs whose cars have not entered yet hold identical states)
    best = (-1.0, 0, 0)
    for t in range(1, fr.shape[0] - 1):
        hv = hs[t].view(fr.shape[1], N, -1)
        d = (hv[:-1] - hv[1:]).abs().amax((1, 2)).masked_fill((fr[t, :-1] != 0) | (fr[t, 1:] != 0), -1.0)
        best = max(best, (float(d.max()), t, int(d.argmax())))
    _, t, env = best
    h = hs[t].clone()
    h[env * N:(env + 1) * N] = hs[t][(env + 1) * N:(env + 2) * N]
    swapped = ref_dict(*step_f64(P, obs(t), h, cs[t], b["s_comm"][t], b["s_alive"][t], fr[t], **kw))
    # a step that starts new episodes, with the resets ignored: the state the last episode left enters the step
    tr_ = next(t for t in range(1, fr.shape[0] - 1) if bool(fr[t].any()))
    unreset = ref_dict(*step_f64(P, obs(tr_), hs[tr_], cs[tr_], b["s_comm"][tr_], b["s_alive"][tr_], None, **kw))
    for what, ts, ref in (("h of env %d + 1 in env %d at step %d" % (env, env, t), t, swapped),
                          ("%d resets of step %d ignored" % (int(fr[tr_].sum()), tr_), tr_, unreset)):
        with pytest.raises(AssertionError) as exc:
            compare("%s, reference with the %s" % (label, what), got(ts), ref)
        print(str(exc.value).splitlines()[0][:300])


@pytest.mark.parametrize("name,B", [("grad_pp_hard_ic3net_h128", 8192), ("grad_tj_hard_ic3net_h128", 4096)])
def test_full_size_every_row_matches_float64(name, B):
    """81 920 rows: 640 tiles, 1280 work items, nine or ten items per CTA.  max_steps 6 over 14 lock-steps: every slot
    starts three episodes, so the fresh branches of the operand preparation and of the epilogue run at full size."""
    tr = make_trainer(name, B, max_steps=6)
    assert tr.grad_kernels
    trainer_rows(tr, 14, "%s B=%d" % (name, B), sensitivity=True)


# ---------------------------------------------------------------------------------------------------- b. row sweep

def sweep_batch(case, N, nsm):
    """Env slots B (N agents each) giving the row / tile / work-item count the case is about."""
    def with_tiles(nt):                                  # R just past nt - 1 tiles: the last tile holds 1..N rows
        return ((nt - 1) * TILE) // N + 1
    if case == "R<64":
        return 63 // N
    if case == "64<R<128":
        return 127 // N
    if case == "R=128k+1":
        return next(b for b in range(1, 1 << 16) if (b * N) % TILE == 1 and b * N > 2 * TILE)
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
    nt, ntp, items, grid = geometry(R)
    ok = {"R<64": R < 64, "64<R<128": 64 < R < 128, "R=128k+1": R % TILE == 1 and nt >= 3,
          "no-padding-tiles": R % TILE == 0 and nt % TILE_PAD == 0,
          "7-padding-tiles": nt % TILE_PAD == 1,
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
    net, a = make_net(N, O, (5, 2), wseed=N, impl=impl)
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
    net, a = make_net(N, O, (5, 2), wseed=7, **kw)
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
    tr = make_trainer(name, B, seed=9, id0=4, max_steps=5)
    trainer_rows(tr, 12, label)


def test_two_pass_rollout_with_resets():
    """comm_passes = 2 in a trainer rollout with episode resets: the recorded values / log-probs and the state entering
    every next step against float64 replayed over the trainer's own (h, c) checkpoints."""
    name = "grad_pp_hard_ic3net_h128"
    tr = make_trainer(name, 1024, seed=21, id0=2, comm_passes=2, max_steps=5, grad_impl="autograd")
    assert tr.policy_net.policy_impl == "tc" and tr.policy_net.is_variant and not tr.grad_kernels
    trainer_rows(tr, 12, "pp hard comm_passes=2 B=1024")


# ---------------------------------------------------------------------------------------------------- d. heads

def direct_step(net, obs, h, c, comm, alive, out, draws=None):
    """ic3_policy_step through the C ABI as CommNetMLP.forward calls it, into the caller's buffers out[h, c, value,
    logp, action] (explicit draws [R, nheads] when given).  Returns the device flag word of the step."""
    from ic3net_b200 import _lib
    lib = _lib.load()
    B = obs.shape[0]
    cfg = net.policy_cfg(B)
    w = net.packed()
    x = torch.empty(B * net.nagents, net.hid_size, device="cuda")
    _lib.check(lib.ic3_encoder_dense(C.byref(cfg), C.byref(w), obs.data_ptr(), x.data_ptr(), _lib.stream()))
    ws, _ = net.workspace(B)
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    io = _lib.PolicyIO(x=x.data_ptr(), h=h.data_ptr(), c=c.data_ptr(), comm_action=_lib.ptr(comm),
                       alive=_lib.ptr(alive), fresh=None, tick=None, draws=_lib.ptr(draws), h_out=out["h"].data_ptr(),
                       c_out=out["c"].data_ptr(), value=out["value"].data_ptr(), logp=out["logp"].data_ptr(),
                       action=_lib.ptr(out.get("action")), workspace=_lib.ptr(ws), err=err.data_ptr())
    _lib.check(lib.ic3_policy_step(C.byref(cfg), C.byref(w), C.byref(io), _lib.stream()))
    torch.cuda.synchronize()
    return int(err.item())


def outputs(R, heads, extra=0):
    """Output buffers with `extra` rows past R, every element a NaN bit pattern (actions: -7)."""
    nan = lambda *s: torch.full(s, 0x7FC0DEAD, dtype=torch.int32, device="cuda").view(torch.float32)
    return dict(h=nan(R + extra, 128), c=nan(R + extra, 128), value=nan(R + extra), logp=nan(R + extra, sum(heads)),
                action=torch.full((R + extra, len(heads)), -7, dtype=torch.int32, device="cuda"))


HEADS = [(5, 2), (2, 2, 2, 1), (9, 2), (5, 5, 5), (3, 4, 2, 5), (9, 8), (16, 15), (8, 8, 8, 7)]


@pytest.mark.parametrize("heads", HEADS, ids=["x".join(map(str, h)) for h in HEADS])
def test_heads_with_explicit_draws(heads):
    """1 + sum(heads) = 8 (fused into the LSTM epilogue, heads_finish_kernel), 9..16 (heads_kernel<16>), 17..32
    (heads_kernel<32>), four heads.  Values / log-probs against float64; actions against the float64 inverse CDF away
    from the CDF edges, and in range everywhere: u24 = 0, u24 = 2^24 - 1 and draws placed on the float64 CDF edges."""
    N, O, B = 7, 61, 300
    R = B * N
    nout = 1 + sum(heads)
    net, a = make_net(N, O, heads, wseed=sum(heads))
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
    out = outputs(R, heads)
    assert direct_step(net, *inputs, out, draws=draws) == 0
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
    net, a = make_net(N, O, heads, wseed=11, passes=passes)
    obs, h, c, comm, alive = synthetic(B, N, O, seed=5)
    before = [t.clone() for t in (obs, h, c, comm, alive)]
    out = outputs(R, heads, extra)
    pristine = {k: v.clone() for k, v in out.items()}
    assert direct_step(net, obs, h, c, comm, alive, out,
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
    net, a = make_net(N, O, (5, 2), wseed=13)
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
    out = outputs(R, (5, 2))
    flags = direct_step(net, obs, h, c, comm, alive, out, draws=torch.zeros(R, 2, dtype=torch.int32, device="cuda"))
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
