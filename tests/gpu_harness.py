"""What the GPU tests share: the fixture trainer, the gradient of a recorded batch and the gradient bar, the record
events, the one-stream schedule check, and the per-row comparison of a policy step against float64.

Not a test module: the test files import from here and from nowhere else among the tests, so a default changed here
changes every test that uses it, and a default changed in a test file changes only that file."""
import argparse
import ctypes as C
import functools
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from bptt_ref import LOSS_KEYS, heads_abs_sums, max_rel_err, oracle_grad_sum, returns_and_advantages, tj_record_obs
from ff_oracle import ff_oracle, records_reference as ff_records_reference
from helpers import finish_args, load_golden, ns
from oracle import philox
from policy_ref import inverse_cdf, params_f64, philox_u24, step_f64

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
PP, TJ = "grad_pp_hard_ic3net_h128", "grad_tj_hard_ic3net_h128"

# ---------------------------------------------------------------------------------------------------- the bars

TOL = 1e-4                  # gradients: per tensor, relative to its largest entry
COL_FLOOR = 1e-6            # encoder columns: floor relative to the whole tensor's largest entry
SUM_FLOOR = 2.0 ** -20      # action heads: floor relative to the sum of |terms| of each entry (16 fp32 ulps)
LOSS_RTOL, LOSS_ATOL = 2e-4, 1e-3
ROW_TOL = 1e-5              # policy steps: |gpu - ref| <= ROW_TOL * max(1, |ref|) on every row (DESIGN.md section 2)
MARGIN = 1e-5               # draws closer than this to a CDF edge may flip between fp32 and float64


def sum_tol(N):
    """Per-row bar of comm_mode sum with several passes: S is up to N - 1 times an h, so each pass multiplies the
    error of h by up to N - 1 through the next S (measured 1.1e-5 at N = 10, 1.8e-5 at N = 20, 5.8e-5 at N = 32)."""
    return max(ROW_TOL, 3e-6 * (N - 1))


# ---------------------------------------------------------------------------------------------------- trainers

IC = dict(commnet=False, hard_attn=False, recurrent=True, rnn_type="MLP")          # models.RNN: the IC / IRIC baselines
FF_FAMILIES = {
    "mlp": dict(model="mlp", commnet=False, hard_attn=False),
    "ic3net": dict(model="commnet", commnet=1, hard_attn=1),
    "commnet": dict(model="commnet", commnet=1, hard_attn=0),
}


def lstm_fixture_weights(meta, args):
    """oracle.gen_golden.make_weights: the recurrent CommNet's state_dict (numpy) under the fixture's weight seed."""
    from oracle.gen_golden import make_weights
    return make_weights(meta["weights_seed"], args.num_inputs, args.hid_size, args.naction_heads, args.comm_init)


def fixture_trainer(name, B, seed=808, id0=30, *, model="commnet", init_seed=None, weights=None, windows=False,
                    **over):
    """Trainer on the recorded arguments of golden fixture ``name``: B env slots with Philox streams (seed, id0 + b),
    index observations, eager rollouts, records for the gradient; ``over`` overrides any argument.

    model: 'commnet' (CommNetMLP), 'rnn' (models.RNN), 'mlp' (models.MLP).  init_seed: torch.manual_seed before the
    module is built (its own initialisation); 'fixture' takes the fixture's weight seed.  weights: then loaded into
    it -- 'fixture' for lstm_fixture_weights, or a state_dict of numpy arrays.  windows: full records never fit, so
    the BPTT records are windows."""
    from ic3net_b200 import data, models
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    meta, _ = load_golden(name)
    kw = dict(nenvs=B, seed=seed, env_id0=id0, obs_mode="index", use_graph=False, record_for_grad=True)
    kw.update(over)
    args = ns(meta["args"], **kw)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    if init_seed is not None:
        torch.manual_seed(meta["weights_seed"] if init_seed == "fixture" else init_seed)
    net = {"commnet": CommNetMLP, "rnn": models.RNN, "mlp": models.MLP}[model](args, args.num_inputs)
    if weights is not None:
        sd = lstm_fixture_weights(meta, args) if isinstance(weights, str) and weights == "fixture" else weights
        net.load_state_dict({k: torch.from_numpy(v).float() for k, v in sd.items()})
    tr = Trainer(args, net, env)
    if windows:
        tr.RECORD_BYTES_LIMIT = 0
    return tr


# The trainers of the gradient tests.  LSTM CommNet / IC3Net on the tensor-core step: with the fixture's weights
# (one comm pass), or the module's own initialisation under the fixture's weight seed (any comm_passes).
lstm_trainer = functools.partial(fixture_trainer, policy_impl="tc", grad_impl="kernels", weights="fixture")
passes_trainer = functools.partial(fixture_trainer, policy_impl="tc", grad_impl="kernels", init_seed="fixture",
                                   comm_passes=1, share_weights=False)
# The IC policy (models.RNN, tanh) on the environment of a fixture, the module's own initialisation.
rnn_trainer = functools.partial(fixture_trainer, model="rnn", init_seed="fixture", policy_impl=None, grad_impl="kernels",
                                comm_passes=1, share_weights=False, **IC)


def ff_trainer(name, B, family, grad_impl="kernels_ff", seed=808, id0=30, weights_seed=77, **over):
    """models.MLP or the non-recurrent CommNet / IC3Net (``family`` of FF_FAMILIES), the module's own initialisation."""
    fam = dict(FF_FAMILIES[family])
    kw = dict(fam, ic3net=False, recurrent=False, rnn_type="MLP", policy_impl=None, grad_impl=grad_impl, comm_passes=1,
              share_weights=False, entr=0.01, comm_mask_zero=False, init_seed=weights_seed)
    kw.update(over)
    return fixture_trainer(name, B, seed, id0, **kw)


def ff_fixture_trainer(name, B, seed, id0, **over):
    """kernels_ff trainer on the arguments and weights of reference fixture ``name`` (tests/golden/gradff_*):
    (trainer, state_dict, meta, z, model)."""
    from ff_oracle import make_weights
    meta, z = load_golden(name)
    a = meta["args"]
    model = "commnet" if a["commnet"] else "mlp"
    sd = make_weights(meta["weights_seed"], meta["obs_dim"], a["hid_size"], meta["heads"], a.get("comm_init", "uniform"),
                      model, int(a["comm_passes"]), bool(a["share_weights"]))
    kw = dict(policy_impl=None, grad_impl="kernels_ff")
    kw.update(over)
    tr = fixture_trainer(name, B, seed, id0, model=model, weights=sd, **kw)
    assert not tr.args.recurrent and tr.grad_ff
    return tr, sd, meta, z, model


def rnn_fixture_trainer(name, B, seed, id0, **over):
    """Kernel trainer on the arguments and weights of reference fixture ``name`` (tests/golden/gradrnn_*):
    (trainer, state_dict, meta, z)."""
    from rnn_oracle import make_weights
    meta, z = load_golden(name)
    sd = make_weights(meta["weights_seed"], meta["obs_dim"], meta["args"]["hid_size"], meta["heads"])
    tr = rnn_trainer(name, B, seed=seed, id0=id0, weights=sd, **over)
    assert tr.grad_kernels and tr.grad_impl == "kernels"
    assert tr.policy_net.policy_impl == (over.get("policy_impl") or "simt")
    return tr, sd, meta, z


def random_args(geometry, **over):
    """Arguments of the reference's --random baseline (models.Random); geometry: BASELINE.json configs[1] ('c2') or
    configs[4] ('c5'), or None."""
    d = dict(hid_size=128, recurrent=False, rnn_type="MLP", commnet=False, ic3net=False, random=True, hard_attn=False,
             comm_action_one=False, comm_mode="avg", comm_passes=1, comm_mask_zero=False, share_weights=False,
             batch_size=500, lrate=1e-3, gamma=1.0, mean_ratio=1.0, normalize_rewards=False, value_coeff=0.01, entr=0.0,
             nenemies=1, no_stay=False, moving_prey=False, enemy_comm=False, mode="mixed", vocab_type="bool",
             add_rate_min=0.05, add_rate_max=0.2, curr_start=0, curr_end=0, difficulty="easy", seed=11, env_id0=0,
             obs_mode="index", use_graph=False, detach_gap=10000, advantages_per_action=False)
    d.update(RANDOM_GEOMETRY[geometry] if geometry else {})
    d.update(over)
    a = argparse.Namespace(**d)
    a.nfriendly = a.nagents
    return a


# BASELINE.json configs[1] and configs[4] (bench.py WORKLOADS pp_hard_ic3net / tj_hard_ic3net), with --random
RANDOM_GEOMETRY = {
    "c2": dict(env_name="predator_prey", nagents=10, dim=20, vision=1, max_steps=80, nenvs=8192, mode="mixed"),
    "c5": dict(env_name="traffic_junction", nagents=20, dim=18, vision=0, max_steps=80, nenvs=4096,
               difficulty="hard", add_rate_min=0.02, add_rate_max=0.05, curr_start=250, curr_end=1250),
}


def random_trainer(args):
    """(models.Random, Trainer) on ``args`` (random_args)."""
    from ic3net_b200 import data, models
    from ic3net_b200.trainer import Trainer
    env = data.init(args.env_name, args)
    finish_args(args, env)
    torch.manual_seed(args.seed)
    net = models.Random(args, args.num_inputs)
    return net, Trainer(args, net, env)


def variant_net(meta, z, policy_impl=None):
    """(args, policy module) of a var_* forward fixture: the reference's state_dict loaded key for key."""
    from ic3net_b200 import models
    from ic3net_b200.comm import CommNetMLP
    a = argparse.Namespace(**meta["args"])
    a.naction_heads, a.continuous = list(meta["heads"]), False
    a.policy_impl = policy_impl
    cls = {"commnet": CommNetMLP, "mlp": models.MLP, "rnn": models.RNN}[meta["model"]]
    net = cls(a, meta["obs_dim"])
    sd = {k[3:]: torch.from_numpy(z[k]).float() for k in z.files if k.startswith("sd_")}
    assert set(net.state_dict().keys()) == set(sd.keys()), (sorted(net.state_dict().keys()), sorted(sd.keys()))
    net.load_state_dict(sd)                               # reference checkpoints load key for key
    return a, net


def close(a, b, tol=ROW_TOL):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.all(np.abs(a - b) <= tol * np.maximum(1.0, np.abs(b)))


# ---------------------------------------------------------------------------------------------------- policy steps

TC_TILE, TC_TILE_PAD = 128, 8   # lstm_tc_kernel: rows per tile; tiles are padded to a multiple of 8 (csrc/policy_tc.cu)
TIE = 1e-5                      # greedy rows whose top two float64 logits are closer than this are exempt


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def tc_geometry(R):
    """(tiles, padded tiles, work items, CTAs) of lstm_tc_kernel for R rows: one item per (tile, 64-unit column half),
    a persistent grid of min(items, SMs) CTAs (one resident CTA per SM)."""
    nt = -(-R // TC_TILE)
    ntp = -(-nt // TC_TILE_PAD) * TC_TILE_PAD
    return nt, ntp, 2 * ntp, min(2 * ntp, sms())


def tc_where(R):
    """compare_rows' ``where`` for lstm_tc_kernel at R rows: the worst element's row, 128-row tile, warpgroup, column
    half, work item and CTA."""
    _, _, items, grid = tc_geometry(R)

    def at(r, col, k):
        tile, wg = r // TC_TILE, (r % TC_TILE) // 64
        if k in ("h", "c"):      # hidden unit `col` belongs to the column half col // 64
            half = col // 64
            item = 2 * tile + half
            return "row %d col %d: tile %d, warpgroup %d, column half %d, item %d, CTA %d (of %d, %d items)" % (
                r, col, tile, wg, half, item, item % grid, grid, items)
        return "row %d col %d: tile %d, warpgroup %d, items %d/%d, CTAs %d/%d (of %d)" % (
            r, col, tile, wg, 2 * tile, 2 * tile + 1, (2 * tile) % grid, (2 * tile + 1) % grid, grid)
    return at


def ref_dict(h, c, value, logps):
    return dict(h=h, c=c, value=value, logp=torch.cat(logps, -1))


def policy_args(N, heads, hard_attn=True, comm_mode="avg", comm_mask_zero=False, passes=1, share=False, impl="tc"):
    return argparse.Namespace(nagents=N, hid_size=128, comm_passes=passes, recurrent=True, rnn_type="LSTM",
                              continuous=False, naction_heads=list(heads), comm_mask_zero=comm_mask_zero,
                              comm_mode=comm_mode, hard_attn=hard_attn, comm_init="uniform", share_weights=share,
                              seed=0, env_id0=0, commnet=True, policy_impl=impl)


def make_lstm_net(N, O, heads, wseed=3, **kw):
    """CommNetMLP with the weights of make_weights (one comm pass) or, with comm_passes > 1, its own seeded init."""
    from ic3net_b200.comm import CommNetMLP
    from oracle.gen_golden import make_weights
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


def lstm_direct_step(net, obs, h, c, comm, alive, out, draws=None):
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


def lstm_outputs(R, heads, extra=0):
    """Output buffers with `extra` rows past R, every element a NaN bit pattern (actions: -7)."""
    nan = lambda *s: torch.full(s, 0x7FC0DEAD, dtype=torch.int32, device="cuda").view(torch.float32)
    return dict(h=nan(R + extra, 128), c=nan(R + extra, 128), value=nan(R + extra), logp=nan(R + extra, sum(heads)),
                action=torch.full((R + extra, len(heads)), -7, dtype=torch.int32, device="cuda"))


def rows_trainer(name, B, seed=5, id0=0, **over):
    """Trainer (tensor-core policy, index observations, records for the gradient) on fixture ``name``'s arguments and
    weights.  With the BPTT kernels the records hold every step's (h, c) (rec_h / rec_c); otherwise grad_window = 1
    checkpoints (h, c) before every step (ck_h / ck_c)."""
    one_pass = int(over.get("comm_passes", load_golden(name)[0]["args"]["comm_passes"])) == 1
    return fixture_trainer(name, B, seed, id0, policy_impl="tc", grad_window=1, init_seed="fixture",
                           weights="fixture" if one_pass else None, **over)


def trainer_rows(tr, T, label, sensitivity=False, where=None):
    """One rollout of T lock-steps, then every row of every step against step_f64 from the recorded state entering the
    step, the recorded observation state and masks.  Recorded actions are recomputed from the reference's log-probs
    with the trainer's own Philox draws.  where: compare_rows' naming of a failing element (default: lstm_tc_kernel's
    work decomposition).  Returns {output: worst error}."""
    e, args = tr.env.env, tr.args
    B, N = e.nenvs, args.nagents
    R = B * N
    where = where or tc_where(R)
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
        compare_rows("%s step %d" % (label, t), got, ref, worst, where=where)
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
        show_sensitivity(tr, P, obs, hs, cs, kw, label, where)
    return worst


def show_sensitivity(tr, P, obs, hs, cs, kw, label, where):
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
            compare_rows("%s, reference with the %s" % (label, what), got(ts), ref, where=where)
        print(str(exc.value).splitlines()[0][:300])


def rnn_step_f64(sd, x_or_obs, h, fresh, N, encoded=False):
    """h' = tanh(affine1(obs) + affine2(h)), value, log-probs in float64 (models.py:83-91); fresh slots enter with h = 0."""
    from ic3net_b200 import bptt
    f64 = torch.float64
    P = {k: v.detach().to("cuda", f64) for k, v in sd.items()}
    h = h.to(f64)
    if fresh is not None:
        h = h.masked_fill(fresh.bool().repeat_interleave(N).unsqueeze(1), 0.0)
    x = x_or_obs.to(f64) if encoded else bptt.encode({"encoder.weight": P["affine1.weight"],
                                                      "encoder.bias": P["affine1.bias"]}, x_or_obs)
    h2 = torch.tanh(x + h @ P["affine2.weight"].t() + P["affine2.bias"])
    nh = sum(1 for k in P if k.startswith("heads.") and k.endswith(".weight"))
    logp = torch.cat([torch.log_softmax(h2 @ P["heads.%d.weight" % m].t() + P["heads.%d.bias" % m], -1)
                      for m in range(nh)], -1)
    return dict(h=h2, value=(h2 @ P["value_head.weight"].t() + P["value_head.bias"])[:, 0], logp=logp)


def rnn_net(N, O, heads, impl, wseed=3, H=128):
    from ic3net_b200 import models
    a = argparse.Namespace(nagents=N, hid_size=H, comm_passes=1, recurrent=True, rnn_type="MLP", continuous=False,
                           naction_heads=list(heads), comm_mask_zero=False, comm_mode="avg", hard_attn=False,
                           comm_init="uniform", share_weights=False, seed=0, env_id0=0, commnet=False, policy_impl=impl)
    torch.manual_seed(wseed)
    return models.RNN(a, O)


def gates_f64(B, N, comm, alive, fresh, hard, avg):
    """(g [B, N, 1], den [B, 1, 1]) of the gated mean (comm.py:102-107,171-175,194-196; trainer.py:45-51)."""
    dev = "cuda"
    fr = (fresh.bool() if fresh is not None else torch.zeros(B, dtype=torch.bool, device=dev)).unsqueeze(1)
    al = alive.double() if alive is not None else torch.ones(B, N, dtype=torch.float64, device=dev)
    al = torch.where(fr, torch.ones_like(al), (al != 0).double())
    n_alive = al.sum(1, keepdim=True)
    g = al * (torch.where(fr, torch.zeros_like(al), (comm != 0).double()) if hard else 1.0)
    one = torch.ones_like(n_alive)
    den = torch.where(n_alive > 1, n_alive - 1, one) if avg else one
    return g.unsqueeze(-1), den.unsqueeze(-1)


def gated_mean(h, g, den):
    """S[k] = g[k] sum_{j != k} g[j] h[j] / den, h [B, N, H]."""
    return g * ((g * h).sum(1, keepdim=True) - g * h) / den


def ff_step_f64(net, x, B, comm=None, alive=None, fresh=None, passes=None):
    """x~ = tanh(x); per pass h = tanh(x~ + C_p(S_p) + f_p(h)); value and log-probs, in float64 (comm.py:127-129,179-239,
    models.py:23-36).  Returns h' of every pass too."""
    w = net._kernel_weights()
    d = lambda t: t.detach().to("cuda", torch.float64)
    cfg = net.policy_cfg(B)
    N, P = net.nagents, passes or max(1, int(cfg.passes))
    xt = torch.tanh(x.double())
    h, hs = xt, []
    g, den = gates_f64(B, N, comm, alive, fresh, bool(cfg.hard_attn), bool(cfg.comm_avg))
    for p in range(P):
        cw, cb = d(w["c_w"][min(p, len(w["c_w"]) - 1)]), d(w["c_b"][min(p, len(w["c_b"]) - 1)])
        z = xt + cb + h @ d(w["f_w"][p]).t() + d(w["f_b"][p])
        if not cfg.comm_mask_zero:
            z = z + (gated_mean(h.view(B, N, -1), g, den).reshape(B * N, -1) @ cw.t())
        h = torch.tanh(z)
        hs.append(h)
    logp = torch.cat([torch.log_softmax(h @ d(hw).t() + d(hb), -1) for hw, hb in zip(w["head_w"], w["head_b"])], -1)
    return dict(h=h, value=(h @ d(w["value_w"]).t() + d(w["value_b"]))[:, 0], logp=logp), hs


def ff_net(N, heads, impl, family="ic3net", passes=1, share=False, mode="avg", wseed=3, H=128, O=61):
    from ic3net_b200 import models
    from ic3net_b200.comm import CommNetMLP
    a = argparse.Namespace(nagents=N, hid_size=H, comm_passes=passes, recurrent=False, rnn_type="MLP", continuous=False,
                           naction_heads=list(heads), comm_mask_zero=False, comm_mode=mode,
                           hard_attn=family == "ic3net", comm_init="uniform", share_weights=share, seed=0, env_id0=0,
                           commnet=family != "mlp", policy_impl=impl)
    torch.manual_seed(wseed)
    return (models.MLP if family == "mlp" else CommNetMLP)(a, O)


def ff_direct_step(net, x, B, out, comm=None, alive=None, fresh=None, draws=None, passes=None):
    """ic3_policy_step as the trainer calls it (the policy's packed weights and workspace), into the caller's buffers;
    returns the device flag word."""
    from ic3net_b200 import _lib
    lib = _lib.load()
    cfg, w = net.policy_cfg(B), net.packed()
    if passes is not None:
        cfg.passes = passes
    ws, _ = net.workspace(B)
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    io = _lib.PolicyIO(x=x.data_ptr(), h=None, c=None, comm_action=_lib.ptr(comm), alive=_lib.ptr(alive),
                       fresh=_lib.ptr(fresh), tick=None, draws=_lib.ptr(draws), h_out=out["h"].data_ptr(), c_out=None,
                       value=out["value"].data_ptr(), logp=out["logp"].data_ptr(), action=_lib.ptr(out.get("action")),
                       workspace=_lib.ptr(ws), err=err.data_ptr())
    _lib.check(lib.ic3_policy_step(C.byref(cfg), C.byref(w), C.byref(io), _lib.stream()))
    torch.cuda.synchronize()
    return int(err.item())


def argmax_check(logits, act, heads, label):
    """act [R, nheads] against the argmax of float64 logits [R, sum(heads)]; rows whose top two logits are within
    TIE * max(1, |logit|) are exempt.  Returns the number of exempt rows."""
    off, exempt = 0, 0
    for k, na in enumerate(heads):
        lg = logits[:, off:off + na]
        want = lg.argmax(1)
        top2 = np.sort(lg, 1)[:, -2:] if na > 1 else np.concatenate([lg - 1, lg], 1)
        near = (top2[:, 1] - top2[:, 0]) < TIE * np.maximum(1.0, np.abs(top2[:, 1]))
        bad = np.nonzero(~near & (want != act[:, k]))[0]
        assert bad.size == 0, "%s head %d: greedy action differs from the float64 argmax at rows %s" % (label, k, bad[:10])
        assert act[:, k].min() >= 0 and act[:, k].max() < na
        exempt += int(near.sum())
        off += na
    return exempt


def head_logits_f64(net, h):
    """Float64 action logits of the heads on hidden state h [R, H] (value head dropped)."""
    w = net._kernel_weights()
    return torch.cat([h.detach().double() @ hw.detach().double().t() + hb.detach().double()
                      for hw, hb in zip(w["head_w"], w["head_b"])], 1)


# ---------------------------------------------------------------------------------------------------- graphed updates

UPDATES = 3                 # updates each graph_update comparison runs
UPDATE_IC = dict(model="rnn", commnet=False, hard_attn=False, recurrent=True, rnn_type="MLP", policy_impl="tc_tanh",
                 comm_passes=1, share_weights=False)
UPDATE_FF = dict(grad_impl="kernels_ff", ic3net=False, recurrent=False, rnn_type="MLP", policy_impl="tc_ff",
                 ff_chunk=7, entr=0.01)


def update_trainer(name, B, graph, ff_chunk=None, **over):
    """Kernel-gradient trainer with graph_update = ``graph`` (lrate 1e-3), the module's own initialisation under the
    fixture's weight seed; ff_chunk sets FF_CHUNK_STEPS."""
    kw = dict(policy_impl="tc", grad_impl="kernels", graph_update=graph, lrate=1e-3, init_seed="fixture")
    kw.update(over)
    tr = fixture_trainer(name, B, **kw)
    if ff_chunk is not None:
        tr.FF_CHUNK_STEPS = ff_chunk
    return tr


def same_stat(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


def cpu(t):
    return t.detach().cpu().numpy()


def episode_trainer(meta, B, obs_mode="index", *, impl=None, seed=None, env_id0=0, use_graph=False, weights=True,
                    **over):
    """(args, env, net, Trainer, float64 weights) on an episode fixture's arguments (``meta``), seed defaulting to the
    fixture's; weights: lstm_fixture_weights loaded into the CommNetMLP (float64 copy returned), else None."""
    from ic3net_b200 import data
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    from oracle import policy as opolicy
    args = ns(meta["args"], nenvs=B, seed=meta["seed"] if seed is None else seed, env_id0=env_id0, obs_mode=obs_mode,
              use_graph=use_graph, policy_impl=impl, **over)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    if impl == "tc" and args.hid_size != 128:
        pytest.skip("tensor-core path is specialised for hid_size 128")
    net = CommNetMLP(args, args.num_inputs)
    p = None
    if weights:
        sd = lstm_fixture_weights(meta, args)
        net.load_state_dict({k: torch.from_numpy(v).float() for k, v in sd.items()})
        p = opolicy.params_to_f64(sd)
    return args, env, net, Trainer(args, net, env), p


# ---------------------------------------------------------------------------------------------------- gradients

def grads_of(tr):
    """compute_grad of the recorded batch from zeroed gradients: ({name: float64 grad}, loss dict)."""
    tr.optimizer.zero_grad(set_to_none=False)
    s = tr.compute_grad(None)
    return {k: p.grad.detach().to(torch.float64).clone() for k, p in tr.policy_net.named_parameters()}, s


def events(tr):
    """How often the batch exercises the record-dependent branches of the backward."""
    b, args = tr._buf, tr.args
    T = b["T"]
    return dict(halted=int((b["valid"] == 0).sum()), fresh=int(b["s_fresh"][1:].sum()) if T > 1 else 0,
                cut=int((((b["s_tep"] + 1) % args.detach_gap) == 0).sum()) if args.detach_gap <= args.max_steps else 0)


def bar_errors(got, ref, sums=None, columns=True):
    """{tensor: error on the TOL scale} of a gradient against a float64 yardstick (<= TOL passes): per tensor the max
    error over TOL of its largest entry, the action heads' entries (keys of ``sums``, heads_abs_sums) also allowed
    SUM_FLOOR of their sum of |terms|, the encoder weight also per input column (TOL of the column's largest entry plus
    COL_FLOOR of the tensor's; not against an fp32 autograd gradient: ``columns``).  A reference tensor that is zero, and a gradient with no reference tensor, must be zero
    exactly (inf otherwise).  Asserts nothing."""
    sums = sums or {}
    errs = {}
    for k, r in ref.items():
        g = got[k].double()
        m = float(r.abs().max())
        if m == 0.0:
            if float(g.abs().max()) != 0.0:
                errs[k] = math.inf
            continue
        if k in sums:
            errs[k] = float(((g - r).abs() / (TOL * m + SUM_FLOOR * sums[k])).max()) * TOL
        else:
            errs[k] = float((g - r).abs().max()) / m
        if columns and r.dim() == 2 and k.endswith(("encoder.weight", "affine1.weight")):
            allowed = TOL * r.abs().amax(0) + COL_FLOOR * m
            errs[k + "[cols]"] = float(((g - r).abs().amax(0) / allowed).max()) * TOL
    for k in got:
        if k not in ref and float(got[k].abs().max()) != 0.0:     # hidd_encoder: not part of the forward
            errs[k] = math.inf
    return errs


def assert_within_bar(got, ref, sums, label, gloss=None, rloss=None, columns=True):
    """bar_errors within TOL, and the loss sums (when given) within rtol 2e-4, atol 1e-3.  Prints; returns the errors."""
    errs = bar_errors(got, ref, sums, columns)
    worst = max(errs, key=errs.get) if errs else None
    losses = "" if gloss is None else " | losses " + " ".join("%s %.6g/%.6g" % (q, gloss[q], rloss[q]) for q in LOSS_KEYS)
    print("%s: worst %s %.2e | %s%s" % (label, worst, errs.get(worst, 0.0),
                                         " ".join("%s %.1e" % kv for kv in errs.items()), losses))
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    assert not bad, (label, bad)
    if gloss is not None:
        for q in LOSS_KEYS:
            assert np.isclose(gloss[q], rloss[q], rtol=LOSS_RTOL, atol=LOSS_ATOL), (label, q, gloss[q], rloss[q])
    return errs


def trainer_within_bar(tr, got, gloss, ref, rloss, label, columns=True):
    """assert_within_bar of compute_grad against a yardstick of the trainer's batch, heads floor from its records."""
    return assert_within_bar(got, ref, heads_abs_sums(tr), label, gloss, rloss, columns)


def kernels_vs_autograd(tk, ta, label):
    """The same seeded batch differentiated by the kernels (tk) and by autograd (ta): the bar against the fp32 autograd
    gradient.  Returns the errors."""
    assert tk.grad_kernels and not ta.grad_kernels
    tk.run_batch(0)
    ta.run_batch(0)
    assert torch.equal(tk._buf["action"], ta._buf["action"])          # one rollout, two backward passes
    gk, sk = grads_of(tk)
    ga, sa = grads_of(ta)
    return trainer_within_bar(tk, gk, sk, ga, sa, label, columns=False)


def assert_same_grads(a, b):
    """Two (gradient dict, loss dict) results bit for bit."""
    (ga, sa), (gb, sb) = a, b
    assert all(torch.equal(ga[k], gb[k]) for k in ga), [k for k in ga if not torch.equal(ga[k], gb[k])]
    assert sa == sb


# ---------------------------------------------------------------------------------------------------- geometry

def pattern_columns(tr):
    """np: columns of the observation pattern the weight-gradient kernel multiplies (csrc/bptt_tc.cu plan_layout)."""
    e = tr.env.env
    W = 2 * e.vision + 1
    used = e.obs_positions + ((W * W + 4) if tr.is_tj else (2 * W * W + 1))
    return (used + 15) // 16 * 16


def wgrad_split(np_cols, sms):
    """(j0, j1): row-tile subsets of the two feature slices of the weight-gradient kernel (plan_layout)."""
    per_mb = sms // 8
    c0 = 3.0 * (128 + 86)
    c1 = 2.0 * (128 + 0.5 * (np_cols - 256) + 22 if np_cols > 256 else 0.5 * np_cols + 22)
    j0 = min(max(int(per_mb * c0 / (c0 + c1) + 0.5), 1), per_mb - 1)
    return j0, per_mb - j0


def sweep_batch(case, sms, N, np_cols):
    """Env slots B (N agents each) giving the row / tile count the case is about."""
    def with_tiles(nt):                # R just past (nt - 1) tiles: the last tile is ragged
        return ((nt - 1) * 128) // N + 1
    if case == "R<64":
        return 63 // N
    if case == "64<R<128":
        return 127 // N
    if case == "R=128k+2":
        return next(b for b in range(2, 10000) if (b * N) % 128 == 2)
    if case == "gates-2-items":
        return with_tiles(sms // 2 + 1)
    if case == "dgrad-2-tiles":
        return with_tiles(sms + 1)
    if case == "wgrad-uneven":
        j0, j1 = wgrad_split(np_cols, sms)
        return with_tiles(j0 * j1 + 1)
    raise KeyError(case)


# ---------------------------------------------------------------------------------------------------- schedule

def one_stream_schedule(tmp_path, module, func, more_than, timeout=600):
    """``module.func(out_dir)`` (a non-test module under tests/) saves .npy files: run it in this process and in a
    child with IC3_BPTT_OVERLAP=0 (read once per process), which keeps the weight-gradient and look-ahead kernels on
    the caller's stream.  Both must save the same files, more than ``more_than`` of them, equal bit for bit.  Returns
    the file names."""
    import importlib
    mine, child = tmp_path / "overlap", tmp_path / "serial"
    mine.mkdir()
    child.mkdir()
    getattr(importlib.import_module(module), func)(str(mine))
    code = "import sys; sys.path[:0] = [%r, %r]; import %s as m; m.%s(%r)" % (ROOT, TESTS, module, func, str(child))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, IC3_BPTT_OVERLAP="0"), cwd=ROOT,
                       capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stderr[-4000:]
    files = sorted(os.listdir(mine))
    assert files == sorted(os.listdir(child)) and len(files) > more_than, files
    for f in files:
        a, b = np.load(mine / f), np.load(child / f)
        assert np.array_equal(a, b), (f, np.abs(a - b).max())
    return files


SCHEDULE_T = (1, 2, 5)         # the parity-indexed buffer sets: one step, both sets once, odd count reusing set 0


def save_schedule_grads(tr, out_dir):
    """Gradients and losses of compute_grad after cut rollouts of T = 1, 2, 5 steps, as .npy files under out_dir."""
    for T in SCHEDULE_T:
        tr.rollout(T, 0, quota=0)
        got, s = grads_of(tr)
        for k, v in got.items():
            np.save(os.path.join(out_dir, "T%d_%s.npy" % (T, k)), v.cpu().numpy())
        np.save(os.path.join(out_dir, "T%d_losses.npy" % T), np.array([s[q] for q in LOSS_KEYS]))


def schedule_lstm(out_dir):
    """One trainer, 400 envs, 32 tiles."""
    save_schedule_grads(lstm_trainer(PP, 400, seed=13, id0=2), out_dir)


def schedule_passes(out_dir):
    """3 comm passes: odd unit counts."""
    save_schedule_grads(passes_trainer(PP, 400, seed=13, id0=2, comm_passes=3), out_dir)


def schedule_rnn(out_dir):
    save_schedule_grads(rnn_trainer(PP, 400, seed=13, id0=2), out_dir)


def schedule_rnn_tc_tanh(out_dir):
    tr = rnn_trainer(PP, 400, seed=13, id0=2, policy_impl="tc_tanh")
    assert tr.policy_net.policy_impl == "tc_tanh"
    save_schedule_grads(tr, out_dir)


# ---------------------------------------------------------------------------------------------------- per-row bar

def rel_err(got, ref):
    got, ref = got.to(torch.float64), ref.to(torch.float64)
    return ((got - ref).abs() / ref.abs().clamp_min(1.0)).reshape(ref.shape[0], -1)


def at_row(r, col, k):
    return "row %d col %d" % (r, col)


def compare_rows(label, got, ref, worst=None, tol=ROW_TOL, where=at_row):
    """got / ref: dicts of h, c [R, H], value [R], logp [R, A] (any may be absent from got).  Asserts every row within
    tol * max(1, |ref|); a failure names the worst element by where(row, col, output).  Returns {output: max error},
    and keeps the running maxima in ``worst``."""
    errs, msgs = {}, []
    R = ref["value"].shape[0]
    for k in ("h", "c", "value", "logp"):
        if k not in got:
            continue
        e = rel_err(got[k].reshape(R, -1), ref[k].reshape(R, -1))
        errs[k] = float(e.max())
        if worst is not None:
            worst[k] = max(worst.get(k, 0.0), errs[k])
        if not errs[k] <= tol:
            r, col = divmod(int(e.nan_to_num(float("inf")).argmax()), e.shape[1])
            msgs.append("%s: %s max %.3e at %s; %d rows over the bar" % (label, k, errs[k], where(r, col, k),
                                                                       int((~(e <= tol)).any(1).sum())))
    assert not msgs, "\n".join(msgs)
    return errs


# ---------------------------------------------------------------------------------------------------- tanh RNN

class _Float64Policy(object):
    """What policy_forward_torch reads of a policy module -- its variant description and its parameters by kernel role --
    with float64 leaf copies of the parameters in P."""

    def __init__(self, net, P, H, device):
        self._cfg_proto = net._cfg_proto
        z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=device)
        nh = sum(1 for n in P if n.startswith("heads.") and n.endswith(".weight"))
        self.w = dict(enc_w=P["affine1.weight"], enc_b=P["affine1.bias"], f_w=[P["affine2.weight"]],
                      f_b=[P["affine2.bias"]], c_w=[z(H, H)], c_b=[z(H)],        # the frozen zero comm buffers
                      value_w=P["value_head.weight"], value_b=P["value_head.bias"],
                      head_w=[P["heads.%d.weight" % m] for m in range(nh)], head_b=[P["heads.%d.bias" % m] for m in range(nh)])

    def _kernel_weights(self):
        return self.w


def rnn_records_reference(tr):
    """Float64 gradient (dict by name) and loss sums of the batch the kernel trainer ``tr`` recorded, one step at a time
    as tests/bptt_ref.py does: step t re-run from rec_h[t] (fresh rows zero) by trainer.policy_forward_torch on float64
    copies of the parameters, the step's loss terms (trainer.py:186-220) differentiated by autograd, the gradient w.r.t.
    h'_t from the later steps dropped at detach cuts.  The loss reads the recorded values and log-probs, as the kernels'
    heads backward does: each enters as  y - y.detach() + recorded,  the recorded number with the float64 step's
    derivative."""
    from ic3net_b200.trainer import policy_forward_torch
    b, args, net, e = tr._buf, tr.args, tr.policy_net, tr.env.env
    assert tr.grad_kernels and "rec_h" in b and "rec_c" not in b
    T, B, N, H = b["T"], e.nenvs, args.nagents, args.hid_size
    R = B * N
    f64 = torch.float64
    ret, adv = returns_and_advantages(tr)
    ret, adv = ret.to(f64).reshape(T, R), adv.to(f64).reshape(T, R)
    P = {n: p.detach().to(f64).requires_grad_(True) for n, p in net.named_parameters()}
    G = {n: torch.zeros_like(p) for n, p in P.items()}
    pol = _Float64Policy(net, P, H, e.device)
    heads = list(args.naction_heads)
    detach = int(args.detach_gap) if int(args.detach_gap) <= int(args.max_steps) else 0
    dh = torch.zeros(R, H, dtype=f64, device=e.device)
    ones = torch.ones(B, N, dtype=f64, device=e.device)        # no communication: the gates do not enter the step
    tot = dict.fromkeys(LOSS_KEYS, 0.0)
    for t in reversed(range(T)):
        frow = b["s_fresh"][t].bool().repeat_interleave(N).unsqueeze(1)
        h0 = b["rec_h"][t].to(f64).requires_grad_(True)
        h = torch.where(frow, torch.zeros_like(h0), h0)
        if tr.is_tj:
            x = F.linear(tj_record_obs(tr, t, 0, B).reshape(R, -1).to(f64), P["affine1.weight"], P["affine1.bias"])
        else:
            idx, val = tr._pp_sparse_obs(b["s_loc"][t])
            x = (F.embedding_bag(idx, P["affine1.weight"].t().contiguous(), per_sample_weights=val.to(f64), mode="sum")
                 + P["affine1.bias"])
        h2, _, value, logps = policy_forward_torch(pol, x, h, None, ones, ones.sum(1, keepdim=True))
        # the step's loss terms (trainer.py:186-220) on the recorded outputs
        alive = b["ralive"][t].reshape(R).to(f64)
        vmask = b["valid"][t].to(f64).repeat_interleave(N)
        act = b["action"][t].long().reshape(R, -1)
        lp_rec = b["logp"][t].reshape(R, -1).to(f64)
        v = value[:, 0]
        v = v - v.detach() + b["value"][t].reshape(R).to(f64)
        lp_taken = torch.zeros(R, dtype=f64, device=e.device)
        ent = torch.zeros((), dtype=f64, device=e.device)
        off = 0
        for m, na in enumerate(heads):
            lp = logps[m] - logps[m].detach() + lp_rec[:, off:off + na]
            lp_taken = lp_taken + lp.gather(1, act[:, m:m + 1]).squeeze(1)             # utils.py:42-46
            ent = ent - (lp * lp.exp() * vmask.unsqueeze(1)).sum()
            off += na
        a_loss = (-adv[t] * lp_taken * alive).sum()
        v_loss = ((v - ret[t]) ** 2 * alive).sum()
        loss = a_loss + args.value_coeff * v_loss
        if args.entr > 0:
            loss = loss - args.entr * ent
        tot["action_loss"] += float(a_loss)
        tot["value_loss"] += float(v_loss)
        tot["entropy"] += float(ent)
        if detach:                                                             # trainer.py:56-60
            cut = (((b["s_tep"][t] + 1) % detach) == 0).repeat_interleave(N).unsqueeze(1)
            dh = torch.where(cut, torch.zeros_like(dh), dh)
        surrogate = loss + (h2 * dh).sum()
        plist = list(P.values())
        gr = torch.autograd.grad(surrogate, plist + [h0], allow_unused=True)
        for (n, _), gp in zip(P.items(), gr[:-1]):
            if gp is not None:
                G[n] += gp
        dh = gr[-1].detach()
    return G, tot


# ---------------------------------------------------------------------------------------------------- one step

OPT_IN = dict(obs_api="handle", forward_grad="kernels")


def handle(tr):
    from ic3net_b200.lazy_obs import LazyObs
    e = tr.env.env
    return LazyObs(e, (e.nenvs, tr.args.nagents, tr.env.observation_dim))


def set_state(tr, t):
    """Put the env state the records hold for step t back into the live env (a handle then describes step t)."""
    e, b = tr.env.env, tr._buf
    for key, attr, _, _ in tr._records:
        getattr(e, attr).copy_(b[key][t])
    e.obs_version += 1


class _Roles(object):
    """Stand-in module for trainer.policy_forward_torch: the policy's kernel-side weights as float64 leaves."""

    def __init__(self, net):
        self._cfg_proto = net._cfg_proto
        self.leaf = {}
        self.w = {k: ([self._conv(t) for t in v] if isinstance(v, list) else self._conv(v))
                  for k, v in net._kernel_weights().items()}

    def _conv(self, t):
        if id(t) not in self.leaf:
            self.leaf[id(t)] = t.detach().double().requires_grad_(isinstance(t, torch.nn.Parameter))
        return self.leaf[id(t)]

    def _kernel_weights(self):
        return self.w


def encode64(tr, roles, w):
    """x = encoder(obs) in float64 from the live env state."""
    e = tr.env.env
    R = e.nenvs * tr.args.nagents
    if tr.is_tj:
        obs = e._get_obs().reshape(R, -1).double()
        return obs @ w["enc_w"].t() + w["enc_b"]
    idx, val = tr._pp_sparse_obs(e.loc)
    return (w["enc_w"].t()[idx] * val.double().unsqueeze(-1)).sum(1) + w["enc_b"]


def one_step(tr, t, seed=0, scale=1.0, spike=None):
    """forward + backward of step t of the trainer's records (env state, (h, c), masks) under random upstream gradients
    times ``scale``; ``spike = (key, v)`` sets the last entry (last row, last column) of upstream gradient ``key``
    ('dh', 'dc', 'dvalue' or 'dlogp') to v.  Returns (kernel gradients by name + 'h' / 'c', float64 gradients, |terms|
    sums of the action heads)."""
    from ic3net_b200.trainer import policy_forward_torch
    net, args, e, b = tr.policy_net, tr.args, tr.env.env, tr._buf
    B, N, H = e.nenvs, args.nagents, args.hid_size
    R = B * N
    lstm = net._cfg_proto["cell"] == 0
    hard = bool(args.hard_attn) and bool(args.commnet)
    set_state(tr, t)
    h = b["rec_h"][t].clone().requires_grad_(True)
    c = b["rec_c"][t].clone().requires_grad_(True) if lstm else None
    comm, alive = b["s_comm"][t].clone(), b["s_alive"][t].clone()
    info = dict(alive_mask=alive)
    if hard:
        info["comm_action"] = comm
    g = torch.Generator(device="cuda").manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    net.zero_grad(set_to_none=True)
    action, value, hid = net([handle(tr), (h, c) if lstm else h], info)
    h2, c2 = hid if lstm else (hid, None)
    assert value.grad_fn is not None and h2.grad_fn is not None and all(a.grad_fn is not None for a in action)
    logp = torch.cat(action, -1).reshape(R, -1)
    up = dict(dlogp=rnd(R, logp.shape[1]) * scale, dvalue=rnd(R) * scale, dh=rnd(R, H) * (0.1 * scale),
              dc=rnd(R, H) * (0.1 * scale))
    if spike is not None:
        up[spike[0]].view(-1)[-1] = spike[1]
    loss = (logp * up["dlogp"]).sum() + (value.reshape(R) * up["dvalue"]).sum() + (h2 * up["dh"]).sum()
    if lstm:
        loss = loss + (c2 * up["dc"]).sum()
    loss.backward()
    got = {n: p.grad.detach().clone() for n, p in net.named_parameters() if p.grad is not None}
    got["h"] = h.grad.detach().clone()
    if lstm:
        got["c"] = c.grad.detach().clone()
    # float64 autograd of the same step
    roles = _Roles(net)
    w = roles.w
    h64 = b["rec_h"][t].double().requires_grad_(True)
    c64 = b["rec_c"][t].double().requires_grad_(True) if lstm else None
    x = encode64(tr, roles, w)
    a64 = alive.double()
    n_alive = a64.sum(1, keepdim=True)
    gate = a64 * comm.double() if hard else a64
    hh, cc, v64, lps = policy_forward_torch(roles, x, h64, c64, gate, n_alive)
    lp64 = torch.cat(lps, -1)
    L = ((lp64 * up["dlogp"].double()).sum() + (v64.reshape(R) * up["dvalue"].double()).sum()
         + (hh * up["dh"].double()).sum())
    if lstm:
        L = L + (cc * up["dc"].double()).sum()
    names = {id(p): n for n, p in net.named_parameters()}
    leaves = [(names[i], t) for i, t in roles.leaf.items() if i in names]
    inputs = [h64] + ([c64] if lstm else []) + [t for _, t in leaves]
    out = torch.autograd.grad(L, inputs)
    ref = {"h": out[0]}
    if lstm:
        ref["c"] = out[1]
    for (n, _), gr in zip(leaves, out[len(inputs) - len(leaves):]):
        ref[n] = gr
    # |terms| of the action heads' gradients: |d logit|^T |h'|
    sums, off = {}, 0
    dl = up["dlogp"].double()
    for m, na in enumerate(args.naction_heads):
        lpm = lp64[:, off:off + na].detach()
        d = dl[:, off:off + na]
        dlogit = (d - lpm.exp() * d.sum(1, keepdim=True)).abs()
        pre = [k for k in ref if k.endswith("heads.%d.weight" % m)][0][:-len("weight")]
        sums[pre + "weight"] = dlogit.t() @ hh.detach().abs()
        sums[pre + "bias"] = dlogit.sum(0)
        off += na
    assert int(b["err"].item()) == 0
    return got, ref, sums


# ---------------------------------------------------------------------------------------------------- windows

def flat_grad(tr):
    """compute_grad of the last rollout from zeroed gradients: (flat gradient buffer, float64 loss sums), copies."""
    tr.optimizer.zero_grad(set_to_none=False)
    losses = tr.compute_grad_device(None).clone()
    g = tr.optimizer.flat_grads.clone()
    assert int(tr._buf["err"].item()) == 0
    return g, losses


def row_mask(tr, t):
    """[B*N] rows of the env slots that were still playing at step t."""
    return tr._buf["valid"][t].bool().repeat_interleave(tr.args.nagents)


def schedule_windows(out_dir):
    """window_vs_full at one-step and ragged windows; saves the window-mode gradients and losses under out_dir."""
    for W in (1, 5):
        out, _ = window_vs_full(PP, 400, W, seed=13, id0=2)
        g, s = out["window"]
        np.save(os.path.join(out_dir, "W%d_grad.npy" % W), g)
        np.save(os.path.join(out_dir, "W%d_losses.npy" % W), s)


def window_vs_full(name, B, W, **over):
    """Full-record and window-record trainers on the same seeded batch: asserts bit-identical rollouts, gradients and
    loss sums, and every recomputed window equal to the full record on the rows of slots still playing.  Returns
    {mode: (flat gradient, losses)} as numpy arrays and the full trainer."""
    tf = lstm_trainer(name, B, grad_window=W, **over)
    tw = lstm_trainer(name, B, grad_window=W, windows=True, **over)
    out = {}
    for tr in (tf, tw):
        tr.run_batch(0)
        g, s = flat_grad(tr)
        out[tr.record_mode] = (g.cpu().numpy(), s.cpu().numpy())
    assert tf.record_mode == "full" and tw.record_mode == "window" and "rec_h" not in tw._buf
    for k in ("action", "valid", "logp", "value", "s_fresh", "s_tep"):
        assert torch.equal(tf._buf[k], tw._buf[k]), k
    T = tw._buf["T"]
    for k in range((T + W - 1) // W):
        wh, wc = tw._recompute_window(k)
        for j in range(wh.shape[0]):
            t = k * W + j
            m = row_mask(tw, t)
            assert torch.equal(wh[j][m], tf._buf["rec_h"][t + 1][m]), (k, j)
            assert torch.equal(wc[j][m], tf._buf["rec_c"][t + 1][m]), (k, j)
        if k + 1 < (T + W - 1) // W:     # the checkpoints are the rollout's state at the window starts
            m = row_mask(tw, (k + 1) * W - 1)
            assert torch.equal(tw._buf["ck_h"][k + 1][m], tf._buf["rec_h"][(k + 1) * W][m]), k
    (gf, sf), (gw, sw) = out["full"], out["window"]
    assert np.array_equal(gf, gw), np.abs(gf - gw).max()
    assert np.array_equal(sf, sw), (sf, sw)
    assert np.isfinite(gf).all() and np.abs(gf).max() > 0
    return out, tf


# ---------------------------------------------------------------------------------------------------- scale swings

SMALL = {PP: 37, TJ: 24}               # 370 / 480 rows: ragged last tiles
SWING = 1e4
GAMMA0 = dict(gamma=0.0, mean_ratio=0.0, normalize_rewards=False)    # advantage of step t from the reward of step t


def step_adv(tr):
    """np [T]: max over rows of |advantage * alive| per step, float64 -- what the heads' d outputs scale with."""
    b = tr._buf
    T = b["T"]
    _, adv = returns_and_advantages(tr)
    a = adv.to(torch.float64).reshape(T, -1) * b["ralive"][:T].reshape(T, -1).to(torch.float64)
    return a.abs().amax(1).cpu().numpy()


def swing(tr, pattern, factor=SWING):
    """Scale the recorded rewards by step: 'even' / 'odd' steps x factor, 'block' the first half / factor and the
    second half x factor.  Asserts the swing of the per-step advantage maxima it was made for."""
    r, T = tr._buf["reward"], tr._buf["T"]
    with torch.no_grad():
        if pattern == "even":
            r[0:T:2] *= factor
        elif pattern == "odd":
            r[1:T:2] *= factor
        else:
            r[:T // 2] /= factor
            r[T // 2:T] *= factor
    # Steps after every slot has halted have no live row (a = 0) and are left out.  Steps whose reward is zero on
    # every row (traffic junction's first step of an episode) keep their advantage, -value, whatever the factor: at
    # least 80% of the neighbouring live pairs (of the second half's live steps) must swing.
    a = step_adv(tr)
    if pattern == "block":
        hi = a[T // 2:]
        ratios = hi[hi > 0] / a[:T // 2].max()
    else:
        lo, hi = np.minimum(a[1:], a[:-1]), np.maximum(a[1:], a[:-1])
        ratios = hi[lo > 0] / lo[lo > 0]
    assert len(ratios) >= T // 4, (pattern, a)
    ratio = np.quantile(ratios, 0.2)
    assert ratio >= 1e3, (pattern, ratio, a)
    return ratio


def finite_and_clean(tr, got, label):
    bad = [k for k, v in got.items() if not torch.isfinite(v).all()]
    assert not bad, (label, "non-finite gradient", bad)
    err = int(tr._buf["err"].item())
    assert err == 0, (label, "error word", hex(err))


def swing_grads(out_dir):
    """Kernel gradients and losses of two swing batches (even steps of predator-prey, odd steps of traffic junction),
    saved under out_dir.  Run in this process and in a child with IC3_BPTT_OVERLAP=0."""
    for name, pattern in ((PP, "even"), (TJ, "odd")):
        tr = lstm_trainer(name, SMALL[name], seed=41, id0=5, **GAMMA0)
        tr.run_batch(0)
        swing(tr, pattern)
        got, s = grads_of(tr)
        finite_and_clean(tr, got, name)
        for k, v in got.items():
            np.save(os.path.join(out_dir, "%s_%s.npy" % (pattern, k)), v.cpu().numpy())
        np.save(os.path.join(out_dir, "%s_losses.npy" % pattern), np.array([s[q] for q in sorted(s)]))


# ---------------------------------------------------------------------------------------------------- tanh RNN checks
# Run by tests/test_gpu_bptt_rnn.py on the SIMT step (policy_impl None) and by tests/test_gpu_rnn_tc.py on 'tc_tanh'.

def rnn_pinned_oracle(name, B, policy_impl):
    """The fixtures' configurations (IC predator-prey with detach_gap cuts, IRIC traffic junction with cars spawning and
    leaving, the predator-prey hard geometry): the kernels against the float64 tanh-RNN oracle replaying every slot
    teacher-forced (tests/rnn_oracle.py; pinned to the unmodified reference by tests/test_oracle_rnn.py), and against
    the float64 backward over the kernel trainer's own records.  B * N is never a multiple of 128: a ragged last tile."""
    from oracle import policy as opolicy
    from rnn_oracle import rnn_oracle
    seed, id0 = 808, 30
    tr, sd, meta, z = rnn_fixture_trainer(name, B, seed, id0, policy_impl=policy_impl)
    assert (B * tr.args.nagents) % 128 != 0
    batch, stat = tr.run_batch(0)
    T, quota = tr.batch_plan()
    got, gloss = grads_of(tr)
    with rnn_oracle():
        want, wstat, nsteps = oracle_grad_sum(tr.args, z, opolicy.params_to_f64(sd), batch.action.cpu().numpy(),
                                              batch.valid.cpu().numpy(), seed, id0, quota, T)
    assert stat["num_steps"] == nsteps
    oracle = {k: torch.as_tensor(want[k], device="cuda") for k in got if want.get(k) is not None and np.any(want[k])}
    assert set(oracle) == set(got), (sorted(oracle), sorted(got))
    ref, rloss = rnn_records_reference(tr)
    for k, r in ref.items():                   # the two float64 yardsticks agree (fp32 records vs float64 rollout)
        assert max_rel_err(r.cpu().numpy(), want[k]) < 1e-5, (name, k)
    label = "%s B=%d %s" % (name, B, events(tr))
    trainer_within_bar(tr, got, gloss, oracle, wstat, label + " vs oracle")
    trainer_within_bar(tr, got, gloss, ref, rloss, label + " vs float64 records")


def rnn_gradient_arrays(name, policy_impl):
    """One slot with the fixture's seed and env id plays the reference's own batch (same episodes, same actions): the
    kernels' loss sums and gradient against the arrays the unmodified reference's compute_grad produced."""
    meta = load_golden(name)[0]
    tr, sd, meta, z = rnn_fixture_trainer(name, 1, meta["seed"], meta["env_id"], policy_impl=policy_impl)
    batch, stat = tr.run_batch(0)
    assert (stat["num_steps"], stat["num_episodes"]) == (meta["num_steps"], meta["num_episodes"])
    got, gloss = grads_of(tr)
    for q in LOSS_KEYS:
        assert np.isclose(gloss[q], meta[q], rtol=LOSS_RTOL, atol=LOSS_ATOL), (q, gloss[q], meta[q])
    sums = heads_abs_sums(tr)
    errs = {}
    for key in z.files:
        if key.startswith("g_"):
            k, ref = key[2:], torch.as_tensor(z[key], device="cuda")
            g = got[k]
        elif key.startswith("gsample_"):
            k = key[8:]
            step = max(1, got[k].numel() // 2048)
            g, ref = got[k].reshape(-1)[::step][:2048], torch.as_tensor(z[key], device="cuda")
            assert np.allclose([float(got[k].sum()), float(got[k].abs().sum())], z["gsum_" + k][:2], rtol=1e-3,
                               atol=1e-6 * float(z["gsum_" + k][1])), key
        else:
            continue
        allowed = TOL * float(ref.abs().max()) + (SUM_FLOOR * sums[k] if k in sums else 0.0)   # heads: stored whole
        errs[k] = float(((g - ref).abs() / allowed).max()) * TOL
    print("%s vs reference arrays: %s" % (name, " ".join("%s %.1e" % kv for kv in errs.items())))
    assert len(errs) == 8 and all(v <= TOL for v in errs.values()), errs


def rnn_full_size(name, B, policy_impl):
    """81 920 rows (640 tiles), the reference batch boundary."""
    tr = rnn_trainer(name, B, seed=5, id0=0, policy_impl=policy_impl)
    assert tr.policy_net.policy_impl == (policy_impl or "simt")
    tr.run_batch(0)
    got, gloss = grads_of(tr)
    ref, rloss = rnn_records_reference(tr)
    trainer_within_bar(tr, got, gloss, ref, rloss, "%s B=%d" % (name, B))


def rnn_run_to_run(policy_impl):
    tr = rnn_trainer(TJ, 300, mean_ratio=0.0, policy_impl=policy_impl)
    assert tr.policy_net.policy_impl == (policy_impl or "simt")
    tr.run_batch(0)
    assert_same_grads(grads_of(tr), grads_of(tr))


def rnn_windows(name, window, policy_impl):
    """Window mode re-runs the index encoder and the policy step from the recorded env state: the same h' bit for bit,
    so the same gradient."""
    tf = rnn_trainer(name, 200, grad_window=window, policy_impl=policy_impl)
    tw = rnn_trainer(name, 200, grad_window=window, windows=True, policy_impl=policy_impl)
    out = {}
    for tr in (tf, tw):
        tr.run_batch(0)
        out[tr.record_mode] = grads_of(tr)
    assert tf.record_mode == "full" and tw.record_mode == "window"
    assert tf.policy_net.policy_impl == tw.policy_net.policy_impl == (policy_impl or "simt")
    assert "rec_c" not in tf._buf and "ck_c" not in tw._buf and "c_abs" not in tw._buf
    assert_same_grads(out["full"], out["window"])


# ---------------------------------------------------------------------------------------------------- non-recurrent checks
# Run by tests/test_gpu_grad_ff.py on the SIMT step (policy_impl None) and by tests/test_gpu_ff_tc.py on 'tc_ff'.

def rollout_and_grad(tr, epoch=0):
    tr.run_batch(epoch)
    return grads_of(tr)


def assert_close(ga, sa, gb, sb, tol=TOL):
    """Kernels against the fp32 autograd recompute: per tensor tol of its largest entry, loss sums rtol 2e-4."""
    assert ga.keys() == gb.keys()
    for k in ga:
        m = float(gb[k].abs().max())
        err = float((ga[k] - gb[k]).abs().max())
        assert err <= tol * max(m, 1e-30), (k, err, m)
    for k in sa:
        assert sa[k] == pytest.approx(sb[k], rel=2e-4, abs=1e-6), k


def check_ff_records(tr, label):
    got, gloss = grads_of(tr)
    ref, rloss, hsum = ff_records_reference(tr)
    assert_within_bar(got, ref, hsum, label, gloss, rloss)
    assert int(tr._buf["err"].item()) == 0
    return got, ref


def ff_pinned_oracle(name, B, policy_impl):
    """Every slot replayed teacher-forced by the float64 oracle of the fixture's policy; B * N never a multiple of 64."""
    from oracle import policy as opolicy
    seed, id0 = 808, 30
    tr, sd, meta, z, model = ff_fixture_trainer(name, B, seed, id0, policy_impl=policy_impl)
    assert (B * tr.args.nagents) % 64 != 0
    batch, stat = tr.run_batch(0)
    T, quota = tr.batch_plan()
    got, gloss = grads_of(tr)
    a = tr.args
    with ff_oracle(model, int(a.comm_passes), bool(a.share_weights)):
        want, wstat, nsteps = oracle_grad_sum(a, z, opolicy.params_to_f64(sd), batch.action.cpu().numpy(),
                                              batch.valid.cpu().numpy(), seed, id0, quota, T)
    assert stat["num_steps"] == nsteps
    oracle = {k: torch.as_tensor(want[k], device="cuda") for k in got}
    ref, rloss, hsum = ff_records_reference(tr)
    for k, r in ref.items():                   # the two float64 yardsticks agree (fp32 records vs float64 rollout);
        # the two-logit comm head's gradient cancels to a small part of its terms, whose fp32 log-probs differ
        allowed = 1e-5 * float(oracle[k].abs().max()) + (SUM_FLOOR * hsum[k] if k in hsum else 0.0)
        assert bool(((r - oracle[k]).abs() <= allowed).all()), (name, k, max_rel_err(r.cpu().numpy(), want[k]))
    assert_within_bar(got, oracle, hsum, gloss=gloss, rloss=wstat, label="%s B=%d vs oracle" % (name, B))
    assert_within_bar(got, ref, hsum, gloss=gloss, rloss=rloss, label="%s B=%d vs float64 records" % (name, B))


def ff_gradient_arrays(name, policy_impl):
    """One slot with the fixture's seed and env id plays the reference's own batch: the kernels' loss sums and gradient
    against the arrays the unmodified reference's compute_grad produced."""
    meta = load_golden(name)[0]
    tr, sd, meta, z, model = ff_fixture_trainer(name, 1, meta["seed"], meta["env_id"], policy_impl=policy_impl)
    batch, stat = tr.run_batch(0)
    assert (stat["num_steps"], stat["num_episodes"]) == (meta["num_steps"], meta["num_episodes"])
    got, gloss = grads_of(tr)
    for q in LOSS_KEYS:
        assert np.isclose(gloss[q], meta[q], rtol=LOSS_RTOL, atol=LOSS_ATOL), (q, gloss[q], meta[q])
    _, _, hsum = ff_records_reference(tr)
    errs = {}
    for key in z.files:
        if key.startswith("g_"):
            k, ref = key[2:], torch.as_tensor(z[key], device="cuda")
            g = got[k]
        elif key.startswith("gsample_"):
            k = key[8:]
            step = max(1, got[k].numel() // 2048)
            g, ref = got[k].reshape(-1)[::step][:2048], torch.as_tensor(z[key], device="cuda")
            assert np.allclose([float(got[k].sum()), float(got[k].abs().sum())], z["gsum_" + k][:2], rtol=1e-3,
                               atol=1e-6 * float(z["gsum_" + k][1])), key
        else:
            continue
        allowed = TOL * float(ref.abs().max()) + (SUM_FLOOR * float(hsum[k].max()) if k in hsum else 0.0)
        errs[k] = float(((g - ref).abs() / allowed).max()) * TOL
    print("%s vs reference arrays: %s" % (name, " ".join("%s %.1e" % kv for kv in errs.items())))
    assert set(errs) == set(got) and all(v <= TOL for v in errs.values()), errs


def ff_full_size(name, family, over, policy_impl):
    """81 920 rows per step at predator-prey hard (8192 slots), 81 920 at traffic-junction hard (4096 slots).
    tests/test_gpu_ff_tc.py runs it on the tc_ff forward."""
    B = 8192 if name == PP else 4096
    tr = ff_trainer(name, B, family, seed=5, id0=0, batch_size=10, policy_impl=policy_impl, **over)
    tr.run_batch(0)
    check_ff_records(tr, "%s B=%d %s %s" % (name, B, family, over))


def ff_chunk_sizes_and_determinism(family, over, policy_impl):
    tr = ff_trainer(PP, 40, family, policy_impl=policy_impl, **over)
    tr.run_batch(0)
    T = tr._buf["T"]
    ref, sref = grads_of(tr)
    again, sagain = grads_of(tr)
    for k in ref:
        assert torch.equal(ref[k], again[k]), k
    assert sref == sagain
    ragged = next(k for k in range(2, T) if T % k)      # a chunk size that does not divide T
    for K in (1, ragged, T + 5):
        tr.FF_CHUNK_STEPS = K
        g, s = grads_of(tr)
        assert tr.ff_chunk_steps == min(K, T)
        assert_close(g, s, ref, sref)
        g2, _ = grads_of(tr)
        for k in g:
            assert torch.equal(g[k], g2[k]), (K, k)


def ff_halted_slots_contribute_nothing(name, family, over, policy_impl):
    """Slots that complete their batch early leave valid = 0 records.  Every record of those slot-steps is changed -- the
    recorded outputs, rewards, post-step alive mask, the step inputs (fresh, comm_action, alive) and the env state (to
    other in-range positions / routes) -- and the gradient and loss sums stay bit-identical, over chunks of one step
    and of several.  Traffic-junction episodes all run to max_steps, so no slot halts early there: the last three
    lock-steps of half the slots are marked valid = 0 instead (both gradients are taken with that marking), and their
    rewards are left alone: those episodes did not end there, so the rewards reach the returns of earlier real steps."""
    tr = ff_trainer(name, 64, family, batch_size=5, policy_impl=policy_impl, **over)
    tr.run_batch(0)
    b = tr._buf
    T, B, N = b["T"], tr.env.env.nenvs, tr.args.nagents
    if tr.is_tj:
        assert bool((b["valid"] == 1).all())
        b["valid"][T - 3:, :B // 2] = 0
    inv = b["valid"] == 0
    assert 0 < int(inv.sum()) < inv.numel()
    for K in (1, 4):
        tr.FF_CHUNK_STEPS = K
        g_all, s_all = grads_of(tr)
        saved = {k: v.clone() for k, v in b.items() if torch.is_tensor(v)}
        b["logp"][inv] = -3.0
        b["value"].view(T, B, N)[inv] = 123.0
        if not tr.is_tj:        # marked slots' episodes go on past the marking: their rewards feed earlier returns
            b["reward"][inv] = 7.0
        b["ralive"][inv] = 1
        b["s_fresh"][inv] = 1 - b["s_fresh"][inv]
        b["s_comm"][inv] = 1
        b["s_alive"][inv] = 1
        if tr.is_tj:
            b["s_tjloc"][inv] = 1
            b["s_tjalive"][inv] = 1
            b["s_tjlast"][inv] = 1
            b["s_tjroute"][inv] = 0
        else:
            b["s_loc"][inv] = torch.randint_like(b["s_loc"][inv], 0, tr.env.env.dim)
        g2, s2 = grads_of(tr)
        for k, v in saved.items():
            b[k].copy_(v)
        for k in g_all:
            assert torch.equal(g_all[k], g2[k]), (K, k)
        assert s_all == s2, K
