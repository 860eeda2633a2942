"""GPU tests of the tanh RNN's tensor-core policy step (csrc/rnn_tc.cu, policy_impl 'tc_tanh': models.RNN with the vanilla
recurrence, the IC / IRIC baselines).

Covered: every row of every step of a rollout with episode resets at the full batch sizes against a float64 step; the
reference's forward fixture and gradient fixtures at the bars of the SIMT path; sampling with explicit draws against the
SIMT path and at the CDF edges; row counts around the 64-row tile and the thresholds of the persistent loop (two CTAs per
SM); rows past R; fresh slots and dead cars; both sides of the fp16 split limit of the weight; the BPTT kernels' gradient
with this forward (float64 records at both full sizes, run-to-run, full / window records and one-stream schedule bit for
bit); CUDA-graph rollouts; the refusals; the command line.

Bar of the forward: |gpu - ref| <= 1e-5 * max(1, |ref|) on h', value and log-probs (DESIGN.md section 2)."""
import argparse
import ctypes as C
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import test_gpu_bptt_rnn as grad_tests
from bptt_ref import tj_record_obs
from helpers import golden_names, load_golden
from oracle import philox
from policy_ref import inverse_cdf, philox_u24

pytestmark = pytest.mark.gpu

TOL, MARGIN, TILE = 1e-5, 1e-5, 64
TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
PP, TJ = grad_tests.PP, grad_tests.TJ


_ic_trainer = grad_tests.make_trainer


def make_trainer(*a, **kw):
    kw.setdefault("policy_impl", "tc_tanh")
    tr = _ic_trainer(*a, **kw)
    assert tr.policy_net.policy_impl == kw["policy_impl"]
    return tr


@pytest.fixture
def tc_tanh_trainers(monkeypatch):
    """The IC trainers of tests/test_gpu_bptt_rnn.py built with policy_impl 'tc_tanh': its checks then run on this
    forward, at the bars the SIMT path meets."""
    monkeypatch.setattr(grad_tests, "make_trainer", functools.partial(make_trainer, policy_impl="tc_tanh"))


def rel_err(got, ref):
    got, ref = got.to(torch.float64), ref.to(torch.float64)
    return ((got - ref).abs() / ref.abs().clamp_min(1.0)).reshape(ref.shape[0], -1)


def compare(label, got, ref, worst=None):
    msgs = []
    R = ref["value"].shape[0]
    for k in got:
        e = rel_err(got[k].reshape(R, -1), ref[k].reshape(R, -1))
        m = float(e.max())
        if worst is not None:
            worst[k] = max(worst.get(k, 0.0), m)
        if not m <= TOL:
            r, col = divmod(int(e.argmax()), e.shape[1])
            msgs.append("%s: %s max %.3e at row %d col %d (tile %d, warp %d); %d rows over the bar" % (
                label, k, m, r, col, r // TILE, (r % TILE) // 16, int((e > TOL).any(1).sum())))
    assert not msgs, "\n".join(msgs)


def step_f64(sd, x_or_obs, h, fresh, N, encoded=False):
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


# ---------------------------------------------------------------------------------------------------- 1. full size

@pytest.mark.parametrize("name,B", [(PP, 8192), (TJ, 4096)])
def test_full_size_every_row_matches_float64(name, B):
    """81 920 rows, 1280 tiles.  max_steps 6 over 14 lock-steps: every slot starts three episodes."""
    tr = make_trainer(name, B, seed=5, id0=0, max_steps=6)
    assert tr.grad_kernels and tr.record_mode == "full"
    e, args = tr.env.env, tr.args
    N, T = args.nagents, 14
    R = B * N
    tick0 = e.tick.clone().to(torch.int64).cpu().numpy()
    tr.rollout(T, 0)
    tr.collect_stat()                                    # raises on a device-side flag
    b = tr._buf
    sd = tr.policy_net.state_dict()
    worst, flips, nfresh = {}, 0, 0
    for t in range(T):
        if tr.is_tj:
            obs = tj_record_obs(tr, t, 0, B).reshape(R, -1).double()
        else:
            idx, val = tr._pp_sparse_obs(b["s_loc"][t])
            obs = (idx, val.double())
        ref = step_f64(sd, obs, b["rec_h"][t], b["s_fresh"][t], N)
        nfresh += int(b["s_fresh"][t].sum())
        compare("%s step %d" % (name, t), dict(h=b["rec_h"][t + 1], value=b["value"][t], logp=b["logp"][t].reshape(R, -1)),
                ref, worst)
        u24 = philox_u24(int(e.cfg.seed), int(e.cfg.env_id0) + np.arange(B)[:, None], (tick0 + t)[:, None],
                         philox.STREAM_ACTION, np.arange(N)[None, :]).reshape(R, 4)
        act = b["action"][t].reshape(R, -1).cpu().numpy()
        off = 0
        for k, na in enumerate(args.naction_heads):
            want, margin = inverse_cdf(ref["logp"][:, off:off + na], u24[:, k])
            bad = np.nonzero((margin > MARGIN) & (want != act[:, k]))[0]
            assert bad.size == 0, (name, t, k, bad[:10])
            flips += int((want != act[:, k]).sum())
            off += na
    assert flips <= 1e-3 * R * T and nfresh > B
    print("%s B=%d: %d rows x %d steps, worst |gpu - ref| / max(1, |ref|): %s; action flips at CDF edges %d" % (
        name, B, R, T, " ".join("%s %.2e" % kv for kv in worst.items()), flips))


# ---------------------------------------------------------------------------------------------------- 2. fixtures

def test_forward_fixture_of_the_reference():
    """var_rnn_tanh (the unmodified reference's models.RNN: its state_dict, inputs, outputs) through models.RNN.forward."""
    from test_gpu_variants import build, close
    meta, z = load_golden("var_rnn_tanh")
    a, net = build(meta, z, "tc_tanh")
    assert net.policy_impl == "tc_tanh"
    B, n, H = z["obs"].shape[0], a.nagents, a.hid_size
    obs = torch.tensor(z["obs"], dtype=torch.float32, device="cuda")
    h = torch.tensor(z["h"], dtype=torch.float32, device="cuda").reshape(B * n, H)
    act, val, h2 = net([obs, h], {})
    torch.cuda.synchronize()
    net.check_errors()
    assert close(val.reshape(B, n).cpu().numpy(), z["value"])
    for k in range(len(meta["heads"])):
        assert close(act[k].cpu().numpy(), z["logp%d" % k]), k
    assert close(h2.reshape(B, n, H).cpu().numpy(), z["h2"])


@pytest.mark.parametrize("name", golden_names("gradrnn_"))
def test_gradient_fixtures_of_the_reference(name, tc_tanh_trainers):
    """One slot replays the reference's own batch (same episodes and actions as the fixture, asserted by the step and
    episode counts and the loss sums): gradient within 1e-4 of the largest entry of the stored arrays; then B = 5 against
    the float64 oracle and the float64 backward over the records."""
    grad_tests.test_kernels_match_reference_gradient_arrays(name)
    grad_tests.test_kernels_match_reference_pinned_oracle(name, 5)


# ---------------------------------------------------------------------------------------------------- direct steps

def rnn_net(N, O, heads, impl, wseed=3, H=128):
    from ic3net_b200 import models
    a = argparse.Namespace(nagents=N, hid_size=H, comm_passes=1, recurrent=True, rnn_type="MLP", continuous=False,
                           naction_heads=list(heads), comm_mask_zero=False, comm_mode="avg", hard_attn=False,
                           comm_init="uniform", share_weights=False, seed=0, env_id0=0, commnet=False, policy_impl=impl)
    torch.manual_seed(wseed)
    return models.RNN(a, O)


def twin_nets(N, O, heads, wseed=3):
    tc, simt = rnn_net(N, O, heads, "tc_tanh", wseed), rnn_net(N, O, heads, "simt", wseed)
    simt.load_state_dict(tc.state_dict())
    return tc, simt


def inputs(B, N, O, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    obs = ((torch.rand(B, N, O, generator=g, device="cuda") < 0.1) *
           torch.randint(1, 4, (B, N, O), generator=g, device="cuda")).float()
    h = torch.rand(B * N, 128, generator=g, device="cuda") * 2 - 1
    alive = torch.randint(0, 2, (B, N), generator=g, device="cuda", dtype=torch.uint8)
    return obs, h, alive


def outputs(R, heads, extra=0):
    nan = lambda *s: torch.full(s, 0x7FC0DEAD, dtype=torch.int32, device="cuda").view(torch.float32)
    return dict(h=nan(R + extra, 128), value=nan(R + extra), logp=nan(R + extra, sum(heads)),
                action=torch.full((R + extra, len(heads)), -7, dtype=torch.int32, device="cuda"))


def direct_step(net, obs, h, out, alive=None, fresh=None, draws=None):
    """ic3_policy_step as the trainer calls it, into the caller's buffers; returns the device flag word."""
    from ic3net_b200 import _lib
    lib = _lib.load()
    B = obs.shape[0]
    cfg, w = net.policy_cfg(B), net.packed()
    x = torch.empty(B * net.nagents, net.hid_size, device="cuda")
    _lib.check(lib.ic3_encoder_dense(C.byref(cfg), C.byref(w), obs.data_ptr(), x.data_ptr(), _lib.stream()))
    ws, _ = net.workspace(B)
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    io = _lib.PolicyIO(x=x.data_ptr(), h=h.data_ptr(), c=None, comm_action=None, alive=_lib.ptr(alive),
                       fresh=_lib.ptr(fresh), tick=None, draws=_lib.ptr(draws), h_out=out["h"].data_ptr(), c_out=None,
                       value=out["value"].data_ptr(), logp=out["logp"].data_ptr(), action=_lib.ptr(out.get("action")),
                       workspace=_lib.ptr(ws), err=err.data_ptr())
    _lib.check(lib.ic3_policy_step(C.byref(cfg), C.byref(w), C.byref(io), _lib.stream()))
    torch.cuda.synchronize()
    return int(err.item()), x


# ---------------------------------------------------------------------------------------------------- 3. sampling

@pytest.mark.parametrize("heads", [(5,), (5, 2), (2, 2, 2, 1), (9, 8), (16, 15)], ids=lambda h: "x".join(map(str, h)))
def test_sampling_with_explicit_draws(heads):
    """Explicit draws: u24 = 0, 2^24 - 1, draws on the float64 CDF edges and random ones.  Actions are in range, equal the
    float64 inverse CDF away from the edges, and equal the SIMT path's wherever both paths' log-probs put the draw on
    the same side of every CDF edge."""
    N, O, B = 7, 61, 300
    R = B * N
    tc, simt = twin_nets(N, O, heads, wseed=sum(heads))
    obs, h, alive = inputs(B, N, O, seed=sum(heads))
    rs = np.random.RandomState(1)
    u24 = rs.randint(0, 1 << 24, size=(R, len(heads))).astype(np.int64)
    rows = np.arange(R)
    u24[rows % 8 == 0] = 0
    u24[rows % 8 == 1] = (1 << 24) - 1
    ref = step_f64(tc.state_dict(), obs.reshape(R, O).double(), h, None, N)
    off = 0
    for k, na in enumerate(heads):
        cdf = np.cumsum(np.exp(ref["logp"][:, off:off + na].cpu().numpy()), -1)
        edge = cdf[rows, rs.randint(0, max(na - 1, 1), R)] * (1 << 24)
        on = (rows % 8 == 2) | (rows % 8 == 3)
        u24[on, k] = np.clip(np.where(rows[on] % 8 == 2, np.floor(edge[on]), np.ceil(edge[on])), 0, (1 << 24) - 1)
        off += na
    draws = torch.as_tensor(u24.astype(np.int32), device="cuda").contiguous()
    o_tc, o_simt = outputs(R, heads), outputs(R, heads)
    assert direct_step(tc, obs, h, o_tc, alive=alive, draws=draws)[0] == 0
    assert direct_step(simt, obs, h, o_simt, alive=alive, draws=draws)[0] == 0
    compare("heads %s" % (heads,), {k: o_tc[k] for k in ("h", "value", "logp")}, ref)
    a_tc, a_simt = o_tc["action"].cpu().numpy(), o_simt["action"].cpu().numpy()
    off = 0
    for k, na in enumerate(heads):
        assert a_tc[:, k].min() >= 0 and a_tc[:, k].max() < na
        want, margin = inverse_cdf(ref["logp"][:, off:off + na], u24[:, k])
        assert not np.any((margin > MARGIN) & (want != a_tc[:, k])), (heads, k)
        w_tc, m_tc = inverse_cdf(o_tc["logp"][:, off:off + na], u24[:, k])
        w_simt, m_simt = inverse_cdf(o_simt["logp"][:, off:off + na], u24[:, k])
        same = (w_tc == w_simt) & (m_tc > MARGIN) & (m_simt > MARGIN)      # the draw clear of every CDF edge of both paths
        assert same.mean() > 0.7 and np.array_equal(a_tc[same, k], a_simt[same, k]), (heads, k)
        off += na


# ---------------------------------------------------------------------------------------------------- 4. row counts

def sweep_rows(case, nsm):
    ctas = 2 * nsm                      # persistent grid: two resident CTAs per SM
    return {"one-row": 1, "tile-1": TILE - 1, "tile+1": TILE + 1, "idle-CTAs": (ctas - 3) * TILE - 5,
            "grid-1": (ctas - 1) * TILE, "grid": ctas * TILE, "grid+1": ctas * TILE + 1,
            "two-tiles": 2 * ctas * TILE - 7, "three-tiles": 2 * ctas * TILE + TILE + 3,
            "three-tiles-all": 3 * ctas * TILE}[case]


@pytest.mark.parametrize("case", ["one-row", "tile-1", "tile+1", "idle-CTAs", "grid-1", "grid", "grid+1", "two-tiles",
                                  "three-tiles", "three-tiles-all"])
def test_row_counts_and_rows_past_R(case):
    """One agent per env, so R is any number: 1 row, a tile minus / plus one row, fewer tiles than CTAs (idle CTAs), one
    tile per CTA exactly and one more, CTAs with two and with three tiles, ragged last tiles.  64 rows past R hold a NaN
    pattern and stay bit for bit; the inputs are not written."""
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    R, O, heads, extra = sweep_rows(case, nsm), 61, (5, 2), 64
    net = rnn_net(1, O, heads, "tc_tanh", wseed=11)
    obs, h, _ = inputs(R, 1, O, seed=R)
    fresh = (torch.arange(R, device="cuda") % 5 == 0).to(torch.uint8)
    before = [t.clone() for t in (obs, h, fresh)]
    out = outputs(R, heads, extra)
    pristine = {k: v.clone() for k, v in out.items()}
    flags, _ = direct_step(net, obs, h, out, fresh=fresh, draws=torch.zeros(R, 2, dtype=torch.int32, device="cuda"))
    assert flags == 0
    bits = lambda t: t.view(torch.int32) if t.dtype == torch.float32 else t
    for k, v in out.items():
        assert torch.equal(bits(v[R:]), bits(pristine[k][R:])), (case, k)
    for x, y in zip((obs, h, fresh), before):
        assert torch.equal(x, y)
    worst = {}
    compare("%s R=%d tiles=%d CTAs=%d" % (case, R, -(-R // TILE), 2 * nsm),
            {k: out[k][:R] for k in ("h", "value", "logp")}, step_f64(net.state_dict(), obs.reshape(R, O).double(), h, fresh, 1),
            worst)
    print(case, R, " ".join("%s %.2e" % kv for kv in worst.items()))


# ---------------------------------------------------------------------------------------------------- 5. masks

def test_fresh_slots_start_from_zero_and_dead_cars_are_stepped_like_simt():
    """A fresh slot's rows of io->h hold NaN: the step must not read them.  The alive mask (dead traffic-junction cars)
    does not enter a step without communication: every row gets value and log-probs, as on the SIMT path."""
    N, O, B, heads = 20, 61, 257, (2,)
    R = B * N
    tc, simt = twin_nets(N, O, heads, wseed=5)
    obs, h, alive = inputs(B, N, O, seed=9)
    fresh = (torch.arange(B, device="cuda") % 3 == 0).to(torch.uint8)
    h[fresh.bool().repeat_interleave(N)] = float("nan")
    o_tc, o_simt = outputs(R, heads), outputs(R, heads)
    draws = torch.full((R, 1), 1 << 23, dtype=torch.int32, device="cuda")
    assert direct_step(tc, obs, h, o_tc, alive=alive, fresh=fresh, draws=draws)[0] == 0
    assert direct_step(simt, obs, h, o_simt, alive=alive, fresh=fresh, draws=draws)[0] == 0
    ref = step_f64(tc.state_dict(), obs.reshape(R, O).double(), h, fresh, N)
    for o in (o_tc, o_simt):
        compare("fresh / dead", {k: o[k] for k in ("h", "value", "logp")}, ref)
    assert int((alive == 0).sum()) > R // 4


# ---------------------------------------------------------------------------------------------------- 6. range

def test_weight_limit_of_the_fp16_split():
    """|affine2.weight| * 256 must stay below 65504: an entry of 255 raises no flag and meets the bar, one of 256 is
    refused with the fp16-range flag (0x200) as a Python exception, not computed with a saturated weight."""
    N, O, B, heads = 10, 61, 40, (5,)
    obs, h, _ = inputs(B, N, O, seed=2)
    h *= 1e-3                                           # keeps 255 h inside tanh's unsaturated range
    for entry, ok in ((255.0, True), (256.0, False)):
        net = rnn_net(N, O, heads, "tc_tanh", wseed=13)
        with torch.no_grad():
            net.affine2.weight[3, 7] = entry
        if ok:
            act, val, h2 = net([obs, h], {})
            torch.cuda.synchronize()
            net.check_errors()
            ref = step_f64(net.state_dict(), obs.reshape(B * N, O).double(), h, None, N)
            compare("|w| 255", dict(h=h2, value=val.reshape(-1), logp=torch.cat(act, -1).reshape(B * N, -1)), ref)
        else:
            net([obs, h], {})
            with pytest.raises(RuntimeError, match="0x200"):
                net.check_errors()


# ---------------------------------------------------------------------------------------------------- 7. gradient

def test_full_size_gradient_matches_float64(tc_tanh_trainers):
    for name, B in ((PP, 8192), (TJ, 4096)):
        grad_tests.test_full_size_gradient_matches_float64(name, B)


def test_gradient_is_bit_identical_run_to_run(tc_tanh_trainers):
    grad_tests.test_repeated_compute_grad_is_bit_identical()


@pytest.mark.parametrize("name,window", [(PP, 4), (TJ, 1)])
def test_windowed_records_are_bit_identical(name, window, tc_tanh_trainers):
    """Window mode re-runs the index encoder and the tc_tanh step: the same h' as the rollout bit for bit."""
    grad_tests.test_windowed_records_are_bit_identical(name, window)


def schedule_grads(out_dir):
    grad_tests.make_trainer = functools.partial(make_trainer, policy_impl="tc_tanh")
    grad_tests.schedule_grads(out_dir)


def test_one_stream_schedule_is_bit_identical(tmp_path):
    mine, child = tmp_path / "overlap", tmp_path / "serial"
    mine.mkdir()
    child.mkdir()
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_rnn_tc as m; m.schedule_grads(%%r)" % (ROOT, TESTS))
    for d, over in ((mine, {}), (child, dict(IC3_BPTT_OVERLAP="0"))):
        r = subprocess.run([sys.executable, "-c", code % str(d)], env=dict(os.environ, **over), cwd=ROOT,
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-4000:]
    files = sorted(os.listdir(mine))
    assert files == sorted(os.listdir(child)) and len(files) > 3
    for f in files:
        assert np.array_equal(np.load(mine / f), np.load(child / f)), f


# ---------------------------------------------------------------------------------------------------- 8. graph

@pytest.mark.parametrize("obs_mode", ["index", "dense"])
def test_graph_rollout_equals_eager(obs_mode):
    recs = []
    for use_graph in (False, True):
        tr = make_trainer(PP, 96, seed=3, id0=1, max_steps=7, obs_mode=obs_mode, use_graph=use_graph)
        tr.rollout(16, 0)
        tr.collect_stat()
        b = tr._buf
        recs.append({k: b[k].clone() for k in ("value", "logp", "action", "reward")})
        recs[-1]["rec_h"] = b["rec_h"][1:].clone()       # row 0 is never written: every slot starts fresh
    for k in recs[0]:
        assert torch.equal(recs[0][k], recs[1][k]), (obs_mode, k)


# ---------------------------------------------------------------------------------------------------- 9. refusals

def test_refusals_and_default():
    from ic3net_b200 import models
    with pytest.raises(NotImplementedError):                       # LSTM cell
        make_trainer(PP, 4, rnn_type="LSTM")
    with pytest.raises(NotImplementedError):                       # models.MLP
        make_trainer(PP, 4, model="mlp")
    with pytest.raises(NotImplementedError):                       # hid_size 64
        make_trainer(PP, 4, hid_size=64, grad_impl="autograd")
    with pytest.raises(NotImplementedError):                       # --commnet (LSTM CommNet and the non-recurrent one)
        make_trainer(PP, 4, model="commnet", commnet=True, rnn_type="LSTM")
    with pytest.raises(NotImplementedError):
        make_trainer(PP, 4, model="commnet", commnet=True, recurrent=False)
    net = rnn_net(3, 29, (5,), None)
    assert isinstance(net, models.RNN) and net.policy_impl == "simt" and net.workspace(4) == (None, None)


# ---------------------------------------------------------------------------------------------------- 10. CLI

def test_command_line(capsys):
    from ic3net_b200 import main as cli
    rc = cli.main(["--env_name", "predator_prey", "--nagents", "3", "--dim", "5", "--max_steps", "20", "--hid_size", "128",
                   "--recurrent", "--policy_impl", "tc_tanh", "--nenvs", "64", "--num_epochs", "1", "--epoch_size", "1",
                   "--batch_size", "40"])
    out = capsys.readouterr().out
    assert rc == 0 and "Epoch" in out, out[-2000:]
