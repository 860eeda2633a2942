"""GPU tests of the tanh RNN's tensor-core policy step (the recurrent form of ff_tc_kernel in csrc/ff_tc.cu, policy_impl
'tc_tanh': models.RNN with the vanilla recurrence, the IC / IRIC baselines).

Covered: every row of every step of a rollout with episode resets at the full batch sizes against a float64 step; the
reference's forward fixture and gradient fixtures at the bars of the SIMT path; sampling with explicit draws against the
SIMT path and at the CDF edges; row counts around the 64-row tile and the thresholds of the persistent loop (two CTAs per
SM); rows past R; fresh slots and dead cars; both sides of the fp16 split limit of the weight; the BPTT kernels' gradient
with this forward (float64 records at both full sizes, run-to-run, full / window records and one-stream schedule bit for
bit); CUDA-graph rollouts; the refusals; the command line.

Bar of the forward: |gpu - ref| <= 1e-5 * max(1, |ref|) on h', value and log-probs (DESIGN.md section 2)."""
import ctypes as C

import numpy as np
import pytest
import torch

from bptt_ref import tj_record_obs
from gpu_harness import (MARGIN, PP, TJ, close, compare_rows, one_stream_schedule, rnn_full_size, rnn_gradient_arrays,
                         rnn_net, rnn_pinned_oracle, rnn_run_to_run, rnn_step_f64, rnn_trainer, rnn_windows, variant_net)
from helpers import golden_names, load_golden
from oracle import philox
from policy_ref import inverse_cdf, philox_u24

pytestmark = pytest.mark.gpu

TILE = 64                   # rows per CTA tile of the tc_tanh step (ff_tc_kernel)


def make_trainer(*a, **kw):
    kw.setdefault("policy_impl", "tc_tanh")
    tr = rnn_trainer(*a, **kw)
    assert tr.policy_net.policy_impl == kw["policy_impl"]
    return tr


def compare(label, got, ref, worst=None):
    """Every row of got against ref at the bar, a failure named by its 64-row tile and 16-row warp."""
    compare_rows(label, got, ref, worst, where=lambda r, col, k: "row %d col %d (tile %d, warp %d)" % (
        r, col, r // TILE, (r % TILE) // 16))


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
        ref = rnn_step_f64(sd, obs, b["rec_h"][t], b["s_fresh"][t], N)
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
    meta, z = load_golden("var_rnn_tanh")
    a, net = variant_net(meta, z, "tc_tanh")
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
def test_gradient_fixtures_of_the_reference(name):
    """One slot replays the reference's own batch (same episodes and actions as the fixture, asserted by the step and
    episode counts and the loss sums): gradient within 1e-4 of the largest entry of the stored arrays; then B = 5 against
    the float64 oracle and the float64 backward over the records."""
    rnn_gradient_arrays(name, "tc_tanh")
    rnn_pinned_oracle(name, 5, "tc_tanh")


# ---------------------------------------------------------------------------------------------------- direct steps

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
    ref = rnn_step_f64(tc.state_dict(), obs.reshape(R, O).double(), h, None, N)
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
            {k: out[k][:R] for k in ("h", "value", "logp")}, rnn_step_f64(net.state_dict(), obs.reshape(R, O).double(), h, fresh, 1),
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
    ref = rnn_step_f64(tc.state_dict(), obs.reshape(R, O).double(), h, fresh, N)
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
            ref = rnn_step_f64(net.state_dict(), obs.reshape(B * N, O).double(), h, None, N)
            compare("|w| 255", dict(h=h2, value=val.reshape(-1), logp=torch.cat(act, -1).reshape(B * N, -1)), ref)
        else:
            net([obs, h], {})
            with pytest.raises(RuntimeError, match="0x200"):
                net.check_errors()


# ---------------------------------------------------------------------------------------------------- 7. gradient

def test_full_size_gradient_matches_float64():
    for name, B in ((PP, 8192), (TJ, 4096)):
        rnn_full_size(name, B, "tc_tanh")


def test_gradient_is_bit_identical_run_to_run():
    rnn_run_to_run("tc_tanh")


@pytest.mark.parametrize("name,window", [(PP, 4), (TJ, 1)])
def test_windowed_records_are_bit_identical(name, window):
    """Window mode re-runs the index encoder and the tc_tanh step: the same h' as the rollout bit for bit."""
    rnn_windows(name, window, "tc_tanh")


def test_one_stream_schedule_is_bit_identical(tmp_path):
    one_stream_schedule(tmp_path, "gpu_harness", "schedule_rnn_tc_tanh", more_than=3)


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
