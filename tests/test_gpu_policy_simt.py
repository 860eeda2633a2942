"""GPU tests of the fp32 SIMT policy step (csrc/policy.cu: policy_step_kernel<H> with heads_for_row<H>, policy_impl
'simt') on EVERY row against float64, at hid_size 32, 64 and 128: the forward of every policy at hid_size 32 / 64, the
default forward of every tanh-cell policy (models.MLP, the non-recurrent CommNet / IC3Net, the tanh RNN of the IC / IRIC
baselines), and comm_passes > 1 / share_weights of the LSTM CommNet / IC3Net below hid_size 128.

Covered:
  1. the tanh yardsticks (gpu_harness.ff_step_f64 and rnn_step_f64) against the reference's own forward
     fixtures var_mlp, var_commnet_nonrec2, var_commnet_nonrec_share (hid_size 32) and var_rnn_tanh, to 1e-10, so
     that the bars below rest on the reference (the LSTM yardstick policy_ref.step_f64 is pinned by
     tests/test_policy_ref.py);
  2. full size from a trainer's own records: every row of every step of a 14-step rollout with three episode starts
     per slot (index observations, so the index encoders at each H too; dead cars on traffic junction) -- the LSTM
     IC3Net at H 64 on predator-prey hard (8192 envs) and traffic-junction hard (4096 envs), at H 128 and 32 on
     predator-prey hard; models.MLP, the non-recurrent IC3Net (1 pass) and CommNet (2 passes) at H 128 and 64 on
     predator-prey hard, the CommNet with 3 shared passes and comm_mode sum on traffic-junction hard; the tanh RNN at
     H 128 and 64; actions against the inverse CDF of the float64 log-probs with the trainer's own Philox draws;
  3. the tile geometry (floor(64 / N) whole envs per CTA, 64 mod N padding rows, a ragged last CTA) for N from 1 to 32
     and one env, one CTA less / exactly / plus one env, and 3001 envs, at H 32, 64 and 128, LSTM and non-recurrent
     IC3Net: CommNetMLP.forward and a direct ic3_policy_step (fresh envs entering with a NaN state, explicit draws,
     sentinel rows past R that must stay untouched);
  4. the variants beyond one CTA at H 32 and 64: LSTM with 2-4 passes with and without share_weights, soft attention,
     comm_mode sum, comm_mask_zero, comm_init zeros; the non-recurrent CommNet / IC3Net with 1-4 passes with and without
     share_weights; models.MLP, the tanh RNN and --enemy_comm (N + 1 agent rows) through a trainer rollout;
  5. heads_for_row<32> / <64> with 1 + sum(heads) from 6 to 32 outputs: explicit draws on the CDF edges, greedy
     actions against the float64 argmax, and exact ties taking the lowest index.

Bar: |gpu - ref| <= 1e-5 * max(1, |ref|) on h', c', value and log-probs (DESIGN.md section 2), except comm_mode sum with
several passes, which takes gpu_harness.sum_tol: S is up to N - 1 times an h, so each pass multiplies the error of
h by up to N - 1 through the next S.  On this kernel too that is what the error follows: 3 shared sum-mode passes with
the 20 traffic-junction agents measured 5.9e-6 (H 128) and 8.2e-6 (H 64) on h', against <= 1.4e-7 for every
avg-mode family.  A failure names the row, env, CTA and its position in the CTA's 64-row tile.  A neighbour env's
state and an ignored reset break the bar (negative controls).

Worst |gpu - ref| / max(1, |ref|) measured on an H100 80GB HBM3 at a 700 W power limit (h' / c' / value / log-probs):
  LSTM IC3Net at full size, H 64: 5.4e-8 / 1.0e-7 / 2.0e-8 / 1.9e-7 on predator-prey hard (8192 envs) and
  7.8e-8 / 1.1e-7 / 2.5e-8 / 1.7e-7 on traffic-junction hard (4096 envs); H 128: 4.7e-8 / 8.6e-8 / 1.3e-8 / 1.8e-7;
  H 32: 7.3e-8 / 9.1e-8 / 3.2e-8 / 2.2e-7;
  the tanh families at full size (MLP, non-recurrent IC3Net, 2-pass CommNet, tanh RNN at H 128 and 64): h' <= 1.4e-7,
  value <= 5.5e-8, log-probs <= 2.2e-7; the 3-pass sum-mode CommNet on traffic-junction hard: 8.2e-6 / - / 8.2e-7 /
  8.1e-7;
  the tile sweep: LSTM 4.2e-7 / 8.8e-7 / 1.5e-7 / 2.8e-7, non-recurrent IC3Net 6.2e-7 / - / 2.1e-7 / 3.2e-7;
  the variants and heads at H 32 / 64: <= 5.2e-7 (c'), every other output <= 4.2e-7.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from bptt_ref import tj_record_obs
from gpu_harness import (MARGIN, PP, ROW_TOL, TJ, argmax_check, compare_rows, ff_direct_step, ff_net, ff_step_f64,
                         ff_trainer, head_logits_f64, policy_args, ref_dict, rnn_net, rnn_step_f64, rnn_trainer,
                         sum_tol, synthetic, trainer_rows, variant_net)
from helpers import load_golden
from oracle import philox
from policy_ref import inverse_cdf, params_f64, philox_u24, step_f64

pytestmark = pytest.mark.gpu

ROWS = 64                   # agent rows per CTA tile of policy_step_kernel
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------------- geometry

def kernel_tiling():
    """The tile rule of csrc/policy.cu that the cases below are chosen for: ROWS agent rows per CTA, floor(ROWS / N)
    whole envs per CTA, ceil(B / that) CTAs.  Read from the source, so that changing it makes the sweep say so instead
    of silently testing other cases."""
    with open(os.path.join(ROOT, "ic3net_b200", "csrc", "policy.cu")) as f:
        src = f.read()
    rows = re.search(r"constexpr int ROWS = (\d+);", src)
    assert rows and int(rows.group(1)) == ROWS, "policy_step_kernel tiles %s rows, the sweep is built for %d" % (
        rows and rows.group(1), ROWS)
    assert "const int epb = ROWS / N;" in src and "(a.cfg.B + epb - 1) / epb" in src, \
        "policy_step_kernel no longer puts floor(ROWS / N) whole envs in each CTA"


def geometry(B, N):
    """(envs per CTA, padding rows of a full CTA, CTAs, envs in the last CTA) of policy_step_kernel."""
    epb = ROWS // N
    ctas = -(-B // epb)
    return epb, ROWS - epb * N, ctas, B - (ctas - 1) * epb


def where(r, B, N):
    epb, _, ctas, last = geometry(B, N)
    env = r // N
    cta = env // epb
    filled = (last if cta == ctas - 1 else epb) * N
    return "row %d (env %d, agent %d): CTA %d of %d, tile row %d of %d filled, %d padding rows" % (
        r, env, r - env * N, cta, ctas, r - cta * epb * N, filled, ROWS - filled)


def at(B, N):
    """compare_rows' ``where`` for policy_step_kernel: the worst element's env, CTA and place in the CTA's tile."""
    return lambda r, col, k: "%s, col %d" % (where(r, B, N), col)


def compare(label, got, ref, B, N, worst=None, tol=ROW_TOL):
    """got / ref: dicts of h, c [R, H], value [R], logp [R, A] (any of them may be absent from got).  Asserts the bar;
    returns {output: max error}."""
    return compare_rows(label, got, ref, worst, tol, where=at(B, N))


def fmt(worst):
    return " ".join("%s %.2e" % kv for kv in worst.items())


# ---------------------------------------------------------------------------------------------------- yardsticks

def reference(net, obs, B, h, c, comm, alive, fresh):
    """Float64 step of net by its family: policy_ref.step_f64 (LSTM cell), rnn_step_f64 (tanh RNN),
    ff_step_f64 (non-recurrent tanh).  obs: dense [R, O] or sparse (index, value), float64."""
    from ic3net_b200 import _lib, bptt
    p, N = net._cfg_proto, net.nagents
    hard = bool(p["hard_attn"])
    if p["cell"] == _lib.CELL_LSTM:
        P = params_f64(net.state_dict(), p["passes"], device="cuda")
        return ref_dict(*step_f64(P, obs, h, c, comm if hard else None, alive, fresh, nagents=N, passes=p["passes"],
                                     hard_attn=hard, comm_mode="avg" if p["comm_avg"] else "sum",
                                     comm_mask_zero=bool(p["comm_mask_zero"])))
    if not p["h_from_x"]:
        return rnn_step_f64(net.state_dict(), obs, h, fresh, N)
    w = net._kernel_weights()
    x = bptt.encode({"encoder.weight": w["enc_w"].detach().double(), "encoder.bias": w["enc_b"].detach().double()}, obs)
    return ff_step_f64(net, x, B, comm if hard else None, alive, fresh)[0]


def sum_mode(net):
    return not net._cfg_proto["comm_avg"] and not net._cfg_proto["comm_mask_zero"] and net._cfg_proto["passes"] > 1


# ---------------------------------------------------------------------------------------------------- 1. yardsticks

@pytest.mark.parametrize("name", ["var_mlp", "var_commnet_nonrec2", "var_commnet_nonrec_share", "var_rnn_tanh"])
def test_tanh_yardsticks_match_the_reference_fixtures(name):
    """The reference's own outputs (float64 modules, its state_dict and inputs) against the tanh yardsticks fed the
    same float64 weights: value, log-probs (and h' of the tanh RNN) within 1e-10."""
    meta, z = load_golden(name)
    K, N, O = z["obs"].shape
    R = K * N
    t = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float64, device="cuda")
    sd = {k[3:]: t(z[k]) for k in z.files if k.startswith("sd_")}
    obs = t(z["obs"]).reshape(R, O)
    if meta["model"] == "rnn":
        ref = rnn_step_f64(sd, obs, t(z["h"]).reshape(R, -1), None, N)
        want = dict(h=t(z["h2"]).reshape(R, -1))
    else:
        _, net = variant_net(meta, z, "simt")
        net.double()
        net.load_state_dict(sd)                           # the fixture's float64 weights, not their float32 rounding
        assert net._kernel_weights()["enc_w"].dtype == torch.float64
        w = net._kernel_weights()
        x = obs @ w["enc_w"].detach().t() + w["enc_b"].detach()
        ref, _ = ff_step_f64(net, x, K, t(z["comm"]) if meta["hard_attn"] else None,
                             t(z["alive"]) if meta["use_alive"] else None, None)
        want = {}
    want.update(value=t(z["value"]).reshape(R),
                logp=torch.cat([t(z["logp%d" % k]).reshape(R, -1) for k in range(len(meta["heads"]))], -1))
    for k, v in want.items():
        err = float(((ref[k].reshape(R, -1) - v.reshape(R, -1)).abs() / v.reshape(R, -1).abs().clamp_min(1.0)).max())
        assert err <= 1e-10, (name, k, err)


# ---------------------------------------------------------------------------------------------------- 2. full size

def check_actions(tr, t, tick0, ref_logp, act):
    """Recorded actions of step t against the inverse CDF of the float64 log-probs with the trainer's Philox draws of
    (seed, env_id0 + b, tick, agent), away from the CDF edges.  Returns the number of rows that differ at an edge."""
    e, heads = tr.env.env, list(tr.args.naction_heads)
    B, N = e.nenvs, tr.args.nagents
    R = B * N
    u24 = philox_u24(int(e.cfg.seed), int(e.cfg.env_id0) + np.arange(B)[:, None], (tick0 + t)[:, None],
                     philox.STREAM_ACTION, np.arange(N)[None, :]).reshape(R, 4)
    act = act.reshape(R, -1).cpu().numpy()
    off, flips = 0, 0
    for k, na in enumerate(heads):
        want, margin = inverse_cdf(ref_logp[:, off:off + na], u24[:, k])
        bad = np.nonzero((margin > MARGIN) & (want != act[:, k]))[0]
        assert bad.size == 0, "step %d head %d: action differs at rows %s" % (t, k, bad[:10])
        flips += int((want != act[:, k]).sum())
        off += na
    return flips


def record_obs(tr, t):
    """Float64 observation of lock-step t from the recorded env state: dense [R, O] (traffic junction) or the sparse
    (index, value) pair (predator-prey)."""
    b, B = tr._buf, tr.env.env.nenvs
    if tr.is_tj:
        return tj_record_obs(tr, t, 0, B).reshape(B * tr.args.nagents, -1).double()
    idx, val = tr._pp_sparse_obs(b["s_loc"][t])
    return idx, val.double()


def record_x(tr, t):
    """x of lock-step t: the index encoder the rollout ran, on the recorded env state (test_gpu_ff_tc.record_inputs at
    any hid_size)."""
    from ic3net_b200 import _lib
    net, e = tr.policy_net, tr.env.env
    cfg, w = net.policy_cfg(e.nenvs), net.packed()
    ecfg, est = tr._record_state(t)
    x = torch.empty(e.nenvs * tr.args.nagents, tr.args.hid_size, device="cuda")
    enc = _lib.load().ic3_tj_encoder_index if tr.is_tj else _lib.load().ic3_pp_encoder_index
    _lib.check(enc(C.byref(ecfg), C.byref(est), C.byref(cfg), C.byref(w), x.data_ptr(), _lib.stream()))
    return x


def outputs(R, H, heads, lstm, extra=0):
    """Output buffers with `extra` rows past R, every element a NaN bit pattern (actions: -7)."""
    nan = lambda *s: torch.full(s, 0x7FC0DEAD, dtype=torch.int32, device="cuda").view(torch.float32)
    out = dict(h=nan(R + extra, H), value=nan(R + extra), logp=nan(R + extra, sum(heads)),
               action=torch.full((R + extra, len(heads)), -7, dtype=torch.int32, device="cuda"))
    if lstm:
        out["c"] = nan(R + extra, H)
    return out


def tanh_rows(tr, T, label, negative=False):
    """trainer_rows for the tanh policies: one rollout of T lock-steps, then every row of every step against float64
    from the records -- the rollout's value / log-probs; h' of the tanh RNN from its (h) checkpoints, h' of the
    non-recurrent step from a direct step on the recorded x (whose value / log-probs must equal the rollout's bit for
    bit); actions against the float64 inverse CDF.  negative: a neighbour env's observation (non-recurrent) or an
    ignored reset (tanh RNN) must break the bar."""
    e, args, net = tr.env.env, tr.args, tr.policy_net
    B, N, H = e.nenvs, args.nagents, args.hid_size
    R = B * N
    heads = list(args.naction_heads)
    assert net.policy_impl == "simt" and not tr.grad_kernels and tr.grad_window == 1
    rnn = not net._cfg_proto["h_from_x"]
    tol = sum_tol(N) if sum_mode(net) else ROW_TOL
    tick0 = e.tick.clone().to(torch.int64).cpu().numpy()
    tr.rollout(T, 0)
    tr.collect_stat()                                    # raises on a device-side flag
    assert int(tr._buf["err"].item()) == 0
    b = tr._buf
    worst, flips, nfresh, ndead = {}, 0, 0, 0
    for t in range(T):
        comm, alive, fresh = b["s_comm"][t], b["s_alive"][t], b["s_fresh"][t]
        obs = record_obs(tr, t)
        hin = b["ck_h"][t] if rnn else None
        ref = reference(net, obs, B, hin, None, comm, alive, fresh)
        got = dict(value=b["value"][t].reshape(R), logp=b["logp"][t].reshape(R, -1))
        if rnn and t + 1 < T:                            # checkpoints hold the state entering steps 0 .. T-1
            got["h"] = b["ck_h"][t + 1]
        elif not rnn:
            out = outputs(R, H, heads, False)
            assert ff_direct_step(net, record_x(tr, t), B, out, comm if tr.hard else None, alive, fresh) == 0
            assert torch.equal(out["value"], got["value"]) and torch.equal(out["logp"], got["logp"]), (label, t)
            got["h"] = out["h"]
        compare("%s step %d" % (label, t), got, ref, B, N, worst, tol)
        flips += check_actions(tr, t, tick0, ref["logp"], b["action"][t])
        nfresh += int(fresh.sum())
        ndead += int((alive == 0).sum())
        if negative and t >= 1 and (not rnn or bool(fresh.any())):
            if rnn:
                what, bad = "%d resets ignored" % int(fresh.sum()), reference(net, obs, B, hin, None, comm, alive, None)
            else:
                # the dense observation of env 0 taken from env 1 (predator-prey: the sparse pairs)
                o2 = tuple(v.clone() for v in obs) if isinstance(obs, tuple) else (obs.clone(),)
                if all(torch.equal(v[:N], v[N:2 * N]) for v in o2):
                    continue                             # envs 0 and 1 see the same: try the next step
                for v in o2:
                    v[:N] = v[N:2 * N]
                o2 = o2 if isinstance(obs, tuple) else o2[0]
                what, bad = "env 1's observation in env 0", reference(net, o2, B, hin, None, comm, alive, fresh)
            with pytest.raises(AssertionError) as exc:
                compare("%s step %d, reference with the %s" % (label, t, what), got, bad, B, N)
            print(str(exc.value).splitlines()[0][:300])
            negative = False
    assert not negative, "no step for the negative control"
    assert flips <= 1e-3 * R * T * len(heads), flips
    assert nfresh > B and (ndead > 0 or not tr.is_tj)
    print("%s: %d rows x %d steps, worst |gpu - ref| / max(1, |ref|): %s; action flips at CDF edges %d" % (
        label, R, T, fmt(worst), flips))
    return worst


def lstm_trainer(name, B, H, **over):
    tr = ff_trainer(name, B, "ic3net", grad_impl="autograd", policy_impl="simt", hid_size=H, recurrent=True,
                         rnn_type="LSTM", grad_window=1, **over)
    assert tr.policy_net.policy_impl == "simt" and tr.policy_net.recurrent and not tr.grad_kernels
    return tr


def tanh_trainer(name, B, family, H, **over):
    kw = dict(grad_impl="autograd", policy_impl="simt", hid_size=H, grad_window=1)
    if family == "rnn":
        return rnn_trainer(name, B, **dict(kw, **over))
    return ff_trainer(name, B, family, **dict(kw, **over))


LSTM_FULL = [(PP, 8192, 64), (TJ, 4096, 64), (PP, 8192, 128), (PP, 8192, 32)]


@pytest.mark.parametrize("name,B,H", LSTM_FULL)
def test_full_size_lstm_every_row_matches_float64(name, B, H):
    """81 920 rows per step, 14 lock-steps with max_steps 6: every slot starts three episodes.  H 64 on both envs also
    shows that a neighbour env's state and an ignored reset break the bar."""
    tr = lstm_trainer(name, B, H, seed=5, id0=0, max_steps=6)
    trainer_rows(tr, 14, "simt LSTM IC3Net H=%d %s B=%d" % (H, name, B), sensitivity=H == 64,
                 where=at(B, tr.args.nagents))


TANH_FULL = [(PP, 8192, fam, H, over) for H in (128, 64)
             for fam, over in (("mlp", {}), ("ic3net", {}), ("commnet", dict(comm_passes=2)), ("rnn", {}))] + \
            [(TJ, 4096, "commnet", H, dict(comm_passes=3, share_weights=True, comm_mode="sum")) for H in (128, 64)]


@pytest.mark.parametrize("name,B,family,H,over", TANH_FULL, ids=lambda v: "-".join("%s%s" % kv for kv in v.items())
                         or "p1" if isinstance(v, dict) else str(v))
def test_full_size_tanh_every_row_matches_float64(name, B, family, H, over):
    """81 920 rows per step, 14 lock-steps with max_steps 6.  H 64 also shows that a neighbour env's observation
    (non-recurrent IC3Net) and ignored resets (tanh RNN) break the bar."""
    tr = tanh_trainer(name, B, family, H, seed=5, id0=0, max_steps=6, **over)
    tanh_rows(tr, 14, "simt %s H=%d %s B=%d %s" % (family, H, name, B, over), negative=H == 64 and
              family in ("ic3net", "rnn"))


# ---------------------------------------------------------------------------------------------------- 3. tile sweep

def lstm_net(N, O, heads, H, wseed=3, comm_init="uniform", **kw):
    """CommNetMLP with the LSTM cell on the SIMT kernel (test_gpu_policy_rows.policy_args at any hid_size), the module's
    own seeded initialisation."""
    from ic3net_b200.comm import CommNetMLP
    a = policy_args(N, heads, impl="simt", **kw)
    a.hid_size, a.comm_init = H, comm_init
    torch.manual_seed(wseed)
    return CommNetMLP(a, O)


def tanh_net(family, N, O, heads, H, wseed=3, passes=1, share=False, mode="avg"):
    if family == "rnn":
        return rnn_net(N, O, heads, "simt", wseed=wseed, H=H)
    return ff_net(N, heads, "simt", family, passes=passes, share=share, mode=mode, wseed=wseed, H=H, O=O)


def direct_step(net, obs, h, c, comm, alive, fresh, out, draws=None, greedy=False):
    """ic3_policy_step on the SIMT kernel as CommNetMLP._step calls it (ic3_encoder_dense, then the step), with fresh
    envs, explicit draws or greedy actions, into the caller's buffers."""
    from ic3net_b200 import _lib
    lib = _lib.load()
    B = obs.shape[0]
    cfg, w = net.policy_cfg(B), net.packed()
    cfg.greedy = int(greedy)
    assert net.policy_impl == "simt" and net.workspace(B) == (None, None)
    x = torch.empty(B * net.nagents, net.hid_size, device="cuda")
    _lib.check(lib.ic3_encoder_dense(C.byref(cfg), C.byref(w), obs.data_ptr(), x.data_ptr(), _lib.stream()))
    io = _lib.PolicyIO(x=x.data_ptr(), h=_lib.ptr(h), c=_lib.ptr(c), comm_action=_lib.ptr(comm), alive=_lib.ptr(alive),
                       fresh=_lib.ptr(fresh), draws=_lib.ptr(draws), h_out=out["h"].data_ptr(), c_out=_lib.ptr(out.get("c")),
                       value=out["value"].data_ptr(), logp=out["logp"].data_ptr(), action=_lib.ptr(out.get("action")))
    _lib.check(lib.ic3_policy_step(C.byref(cfg), C.byref(w), C.byref(io), _lib.stream()))
    torch.cuda.synchronize()


def inputs(net, B, O, seed):
    """test_gpu_policy_rows.synthetic at the net's hid_size (its h, c cut to H columns), and the fresh envs b % 5 == 3."""
    obs, h, c, comm, alive = synthetic(B, net.nagents, O, seed)
    H = net.hid_size
    fresh = (torch.arange(B, device="cuda") % 5 == 3).to(torch.uint8)
    return obs, h[:, :H].contiguous(), c[:, :H].contiguous(), comm, alive, fresh


def run_case(net, B, O, seed, label, worst=None):
    """CommNetMLP.forward on synthetic inputs, then a direct ic3_policy_step of the same inputs with fresh envs (their
    incoming h, c NaN), explicit draws and 64 sentinel rows past R: every row against float64, the actions against
    the float64 inverse CDF away from the edges, the rows past R and the inputs unchanged bit for bit."""
    N, H = net.nagents, net.hid_size
    R = B * N
    heads = list(net.args.naction_heads)
    from ic3net_b200 import _lib
    carries = not net._cfg_proto["h_from_x"]
    lstm = net._cfg_proto["cell"] == _lib.CELL_LSTM
    tol = sum_tol(N) if sum_mode(net) else ROW_TOL
    obs, h, c, comm, alive, fresh = inputs(net, B, O, seed)
    obs64 = obs.reshape(R, -1).double()
    info = {"alive_mask": alive, "comm_action": comm} if net._cfg_proto["hard_attn"] else {"alive_mask": alive}
    if lstm:
        act, val, (h2, c2) = net([obs, (h, c)], info)
        got = dict(h=h2, c=c2, value=val, logp=torch.cat(act, -1))
    elif carries:
        act, val, h2 = net([obs, h], info)
        got = dict(h=h2, value=val, logp=torch.cat(act, -1))
    else:
        act, val = net(obs, info)
        got = dict(value=val, logp=torch.cat(act, -1))
    torch.cuda.synchronize()
    compare(label + " forward", got, reference(net, obs64, B, h, c if lstm else None, comm, alive, None), B, N, worst,
            tol)
    # direct step: fresh envs enter with NaN, which the step must not read
    rows = fresh.bool().repeat_interleave(N)
    hn, cn = (h.clone(), c.clone()) if carries else (None, None)
    if carries:
        hn[rows] = float("nan")
        cn[rows] = float("nan")
    if not lstm:
        cn = None
    u24 = np.random.RandomState(seed).randint(0, 1 << 24, size=(R, len(heads)))
    draws = torch.as_tensor(u24.astype(np.int32), device="cuda")
    extra = 64
    out = outputs(R, H, heads, lstm, extra)
    pristine = {k: v.clone() for k, v in out.items()}
    ins = [t for t in (obs, hn, cn, comm, alive, fresh, draws) if t is not None]
    before = [t.clone() for t in ins]
    direct_step(net, obs, hn, cn, comm, alive, fresh, out, draws)
    bits = lambda t: t.view(torch.int32) if t.dtype == torch.float32 else t
    for k, v in out.items():
        assert torch.equal(bits(v[R:]), bits(pristine[k][R:])), "%s: %s written past row R = %d" % (label, k, R)
    for a, b in zip(ins, before):
        assert torch.equal(bits(a), bits(b)), "%s: an input was written" % label
    ref = reference(net, obs64, B, hn, cn, comm, alive, fresh)
    errs = compare(label + " direct", {k: out[k][:R] for k in ("h", "c", "value", "logp") if k in out}, ref, B, N,
                   worst, tol)
    act = out["action"][:R].cpu().numpy()
    off = 0
    for k, na in enumerate(heads):
        want, margin = inverse_cdf(ref["logp"][:, off:off + na], u24[:, k])
        bad = np.nonzero((margin > MARGIN) & (want != act[:, k]))[0]
        assert bad.size == 0, "%s head %d: action differs at %s" % (label, k, where(int(bad[0]), B, N))
        assert act[:, k].min() >= 0 and act[:, k].max() < na
        off += na
    return errs


SWEEP_N = [1, 2, 3, 5, 7, 10, 13, 20, 21, 22, 31, 32]
MANY = 3001


def sweep_batches(N):
    """{case: env slots B} for N agents: one env, one CTA less one env, one full CTA, one env in a second CTA, and
    MANY envs over many CTAs with a ragged last one."""
    epb = ROWS // N
    cases = {"one-env": 1, "CTA-1env": epb - 1, "CTA": epb, "CTA+1env": epb + 1, "many-CTAs": MANY}
    return {k: v for k, v in cases.items() if k != "CTA-1env" or v > 1}


def sweep_checks(case, B, N):
    """Asserts that B envs of N agents give policy_step_kernel the geometry the case is named for; returns its label."""
    epb, pad, ctas, last = geometry(B, N)
    ok = {"one-env": B == 1 and ctas == 1 and last * N <= ROWS,
          "CTA-1env": ctas == 1 and last == epb - 1 and ROWS - B * N == N + pad,
          "CTA": ctas == 1 and last == epb and ROWS - B * N == pad,
          "CTA+1env": ctas == 2 and last == 1,
          "many-CTAs": ctas >= 10 and 0 < last < epb}[case]
    assert ok, (case, B, N, epb, pad, ctas, last)
    return "%s N=%d B=%d R=%d: %d envs per CTA, %d padding rows, %d CTAs, %d envs in the last" % (
        case, N, B, B * N, epb, pad, ctas, last)


@pytest.mark.parametrize("family", ["lstm", "ic3net"])
@pytest.mark.parametrize("N", SWEEP_N)
@pytest.mark.parametrize("H", [32, 64, 128])
def test_tile_geometry_sweep(H, N, family):
    """Every geometry of sweep_batches on the LSTM IC3Net (one pass) and the non-recurrent IC3Net (two passes)."""
    kernel_tiling()
    O, heads = 61, (5, 2)
    net = lstm_net(N, O, heads, H, wseed=N) if family == "lstm" else \
        tanh_net("ic3net", N, O, heads, H, wseed=N, passes=2)
    worst = {}
    for case, B in sweep_batches(N).items():
        label = "%s H=%d %s" % (family, H, sweep_checks(case, B, N))
        run_case(net, B, O, seed=1000 * N + H + B, label=label, worst=worst)
    print("%s H=%d N=%d: %s" % (family, H, N, fmt(worst)))


def test_the_sweep_fails_on_a_neighbour_state():
    """Negative control of the sweep: the reference fed env 1's state in env 0 breaks the bar."""
    N, O, B, H = 7, 61, 40, 64
    net = lstm_net(N, O, (5, 2), H)
    obs, h, c, comm, alive, _ = inputs(net, B, O, seed=3)
    info = {"alive_mask": alive, "comm_action": comm}
    act, val, (h2, c2) = net([obs, (h, c)], info)
    got = dict(h=h2, c=c2, value=val, logp=torch.cat(act, -1))
    compare("unchanged", got, reference(net, obs.reshape(B * N, -1).double(), B, h, c, comm, alive, None), B, N)
    hs = h.clone()
    hs[:N] = h[N:2 * N]
    with pytest.raises(AssertionError, match="env 0"):
        compare("neighbour", got, reference(net, obs.reshape(B * N, -1).double(), B, hs, c, comm, alive, None), B, N)


# ---------------------------------------------------------------------------------------------------- 4. variants

VAR_B, VAR_N = 301, 10       # 51 CTAs of 6 envs (4 padding rows), 1 env in the last

LSTM_VARIANTS = [dict(passes=p, share=s) for p in (2, 3, 4) for s in (False, True)] + \
                [dict(hard_attn=False), dict(comm_mode="sum"), dict(comm_mask_zero=True), dict(comm_init="zeros"),
                 dict(passes=3, comm_mode="sum", hard_attn=False)]


@pytest.mark.parametrize("kw", LSTM_VARIANTS, ids=["-".join("%s=%s" % i for i in v.items()) for v in LSTM_VARIANTS])
@pytest.mark.parametrize("H", [32, 64])
def test_lstm_variants_beyond_one_cta(H, kw):
    label = "LSTM H=%d %s %s" % (H, kw, sweep_checks("many-CTAs", VAR_B, VAR_N))
    net = lstm_net(VAR_N, 61, (5, 2), H, wseed=H + len(kw), **kw)
    print(label, fmt(run_case(net, VAR_B, 61, seed=H * 7 + 1, label=label)))


TANH_VARIANTS = [(fam, p, s) for fam in ("ic3net", "commnet") for p in (1, 2, 3, 4) for s in (False, True)
                 if p > 1 or not s]


@pytest.mark.parametrize("family,passes,share", TANH_VARIANTS)
@pytest.mark.parametrize("H", [32, 64])
def test_nonrecurrent_variants_beyond_one_cta(H, family, passes, share):
    label = "%s H=%d passes=%d share=%s %s" % (family, H, passes, share, sweep_checks("many-CTAs", VAR_B, VAR_N))
    net = tanh_net(family, VAR_N, 61, (5, 2), H, wseed=passes + 10 * share, passes=passes, share=share)
    print(label, fmt(run_case(net, VAR_B, 61, seed=H + passes, label=label)))


@pytest.mark.parametrize("family", ["mlp", "rnn"])
@pytest.mark.parametrize("H", [32, 64])
def test_mlp_and_tanh_rnn_direct_beyond_one_cta(H, family):
    label = "%s H=%d %s" % (family, H, sweep_checks("many-CTAs", VAR_B, VAR_N))
    net = tanh_net(family, VAR_N, 61, (5,), H, wseed=H)
    print(label, fmt(run_case(net, VAR_B, 61, seed=H + 5, label=label)))


@pytest.mark.parametrize("family", ["mlp", "rnn", "enemy_comm"])
@pytest.mark.parametrize("H", [32, 64])
def test_trainer_rollout_beyond_one_cta(H, family):
    """models.MLP, the tanh RNN (IC) and the LSTM IC3Net with --enemy_comm (the prey is agent row N - 1 of every env)
    in a trainer rollout of 12 lock-steps over 301 slots with episode resets, every row against float64."""
    B, T = 301, 12
    if family == "enemy_comm":
        name = "grad_pp_enemy_ic3net_h128"
        tr = lstm_trainer(name, B, H, seed=9, id0=4, max_steps=5)
        N = tr.args.nagents
        assert N == load_golden(name)[0]["args"]["nfriendly"] + 1 and tr.env.env.nagent_rows == N
        trainer_rows(tr, T, "simt enemy_comm H=%d %s" % (H, sweep_checks("many-CTAs", B, N)), where=at(B, N))
    else:
        tr = tanh_trainer(PP, B, family, H, seed=9, id0=4, max_steps=5)
        tanh_rows(tr, T, "simt %s H=%d %s" % (family, H, sweep_checks("many-CTAs", B, tr.args.nagents)))


# ---------------------------------------------------------------------------------------------------- 5. heads

HEADS = [(5,), (5, 2), (2, 2, 2, 1), (9, 8), (16, 15)]


@pytest.mark.parametrize("heads", HEADS, ids=["x".join(map(str, h)) for h in HEADS])
@pytest.mark.parametrize("H", [32, 64])
def test_heads_with_explicit_draws_and_greedy(H, heads):
    """heads_for_row<H>: 1 + sum(heads) outputs up to 32 (one per lane).  Explicit draws u24 = 0, 2^24 - 1, on the float64
    CDF edges and random: values / log-probs against float64, actions in range and equal to the float64 inverse CDF
    away from the edges.  Greedy from the same inputs: value / log-probs / h' / c' bit-identical, actions the float64
    argmax; two bit-identical largest logits in a head: the lower index."""
    N, O, B = 7, 61, 300
    R = B * N
    net = lstm_net(N, O, heads, H, wseed=sum(heads))
    obs, h, c, comm, alive, fresh = inputs(net, B, O, seed=1 + sum(heads))
    ref = reference(net, obs.reshape(R, O).double(), B, h, c, comm, alive, fresh)
    rs = np.random.RandomState(sum(heads))
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
    label = "H=%d heads %s (%d outputs)" % (H, heads, 1 + sum(heads))
    out = outputs(R, H, heads, True)
    direct_step(net, obs, h, c, comm, alive, fresh, out, draws)
    errs = compare(label, out, ref, B, N)
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
    greedy = outputs(R, H, heads, True)
    direct_step(net, obs, h, c, comm, alive, fresh, greedy, draws, greedy=True)
    for k in ("h", "c", "value", "logp"):
        assert torch.equal(greedy[k], out[k]), (label, k)
    argmax_check(head_logits_f64(net, greedy["h"]).cpu().numpy(), greedy["action"].cpu().numpy(), heads, label)
    # ties: action lo's weights and bias copied to action na - 1, both well above the others
    lows = []
    with torch.no_grad():
        for hw, hb in zip(net._kernel_weights()["head_w"], net._kernel_weights()["head_b"]):
            na = hw.shape[0]
            lo = (na - 1) // 2
            hb[lo] = hb.max() + 10.0
            hw[na - 1], hb[na - 1] = hw[lo], hb[lo]
            lows.append(lo)
    tied = outputs(R, H, heads, True)
    direct_step(net, obs, h, c, comm, alive, fresh, tied, draws, greedy=True)
    assert bool((tied["action"] == torch.tensor(lows, dtype=torch.int32, device="cuda")).all()), (label, lows)
    print(label, fmt(errs))
