"""The BPTT kernels (csrc/bptt_tc.cu) on the tanh RNN without communication: models.RNN with rnn_type 'MLP', the IC and
IRIC baselines (IRIC = IC with mean_ratio 0), which run on the SIMT policy kernel.

Covered:
  - the gradient against a float64 backward over the kernel trainer's own records (h alone): every step re-run in
    float64 from rec_h[t], the heads' backward started from the recorded log-probs and values as the kernels' is, the
    recursion carried step by step; on ragged tiles, at row counts around the thresholds of the tanh, dgrad and
    weight-gradient kernels (from the card's SM count), and at the full batch sizes;
  - a cross-check against the torch-autograd windowed recompute of the same rollout;
  - bit-identical gradients run to run, between the two-stream and the one-stream schedule, between full and windowed
    records;
  - the refusals (tanh cells with communication, models.MLP, the non-recurrent CommNet, a 7x7 window, an observation
    pattern wider than 512 columns) and train_batch end to end.

Bar against float64: that of tests/test_gpu_bptt_kernels.py: per tensor 1e-4 of its largest entry (affine1.weight also
per input column), the action heads also 2^-20 of their sum of |terms|; loss sums rtol 2e-4.  Against autograd: the bar
of tests/test_gpu_bptt_passes.py."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from bptt_ref import LOSS_KEYS, heads_abs_sums, max_rel_err, oracle_grad_sum, returns_and_advantages, tj_record_obs
from helpers import finish_args, golden_names, load_golden, ns

pytestmark = pytest.mark.gpu

TOL = 1e-4
COL_FLOOR = 1e-6
SUM_FLOOR = 2.0 ** -20
TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
PP, TJ = "grad_pp_hard_ic3net_h128", "grad_tj_hard_ic3net_h128"
IC = dict(commnet=False, hard_attn=False, recurrent=True, rnn_type="MLP")


def make_trainer(name, B, seed=808, id0=30, grad_impl="kernels", windows=False, model="rnn", weights_seed=None,
                 state_dict=None, **over):
    """Trainer of the IC policy (models.RNN, tanh) on the environment arguments of fixture ``name`` (overridden by
    ``over``); the module's own initialisation under a fixed seed, so two trainers of the same arguments hold the same
    weights, or ``state_dict`` (numpy arrays) loaded before the Trainer is built."""
    from ic3net_b200 import data, models
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    meta, _ = load_golden(name)
    kw = dict(IC, nenvs=B, seed=seed, env_id0=id0, obs_mode="index", use_graph=False, policy_impl=None,
              record_for_grad=True, grad_impl=grad_impl, comm_passes=1, share_weights=False)
    kw.update(over)
    args = ns(meta["args"], **kw)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    torch.manual_seed(meta["weights_seed"] if weights_seed is None else weights_seed)
    cls = {"rnn": models.RNN, "mlp": models.MLP, "commnet": CommNetMLP}[model]
    net = cls(args, args.num_inputs)
    if state_dict is not None:
        net.load_state_dict({k: torch.from_numpy(v).float() for k, v in state_dict.items()})
    tr = Trainer(args, net, env)
    if windows:
        tr.RECORD_BYTES_LIMIT = 0
    return tr


def grads_of(tr):
    """compute_grad of the recorded batch from zeroed gradients: ({name: float64 grad}, loss dict)."""
    tr.optimizer.zero_grad(set_to_none=False)
    s = tr.compute_grad(None)
    return {k: p.grad.detach().to(torch.float64).clone() for k, p in tr.policy_net.named_parameters()}, s


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


def records_reference(tr):
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


def assert_within_bar(tr, got, gloss, ref, rloss, label):
    sums = heads_abs_sums(tr)
    errs = {}
    for k, r in ref.items():
        m = float(r.abs().max())
        if m == 0.0:                                   # the frozen zero comm buffers are not parameters; nothing else
            assert float(got[k].abs().max()) == 0.0, (label, k)
            continue
        allowed = TOL * m + (SUM_FLOOR * sums[k] if k in sums else 0.0)
        errs[k] = float(((got[k] - r).abs() / allowed).max()) * TOL
    g, r = got["affine1.weight"], ref["affine1.weight"]
    allowed = TOL * r.abs().amax(0) + COL_FLOOR * r.abs().max()
    errs["affine1.weight[cols]"] = float(((g - r).abs().amax(0) / allowed).max()) * TOL
    print("%s: %s | losses %s" % (label, " ".join("%s %.1e" % kv for kv in errs.items()),
                                  " ".join("%s %.6g/%.6g" % (q, gloss[q], rloss[q]) for q in LOSS_KEYS)))
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    assert not bad, (label, bad)
    for q in LOSS_KEYS:
        assert np.isclose(gloss[q], rloss[q], rtol=2e-4, atol=1e-3), (label, q, gloss[q], rloss[q])


def events(tr):
    b, args = tr._buf, tr.args
    return dict(fresh=int(b["s_fresh"][1:].sum()), halted=int((b["valid"] == 0).sum()),
                cut=int((((b["s_tep"] + 1) % args.detach_gap) == 0).sum()) if args.detach_gap <= args.max_steps else 0)


# ---------------------------------------------------------------------------------------------------- the reference

def fixture_trainer(name, B, seed, id0):
    """Kernel trainer on the arguments and weights of reference fixture ``name`` (tests/golden/gradrnn_*)."""
    from rnn_oracle import make_weights
    meta, z = load_golden(name)
    sd = make_weights(meta["weights_seed"], meta["obs_dim"], meta["args"]["hid_size"], meta["heads"])
    tr = make_trainer(name, B, seed=seed, id0=id0, state_dict=sd)
    assert tr.grad_kernels and tr.grad_impl == "kernels"
    return tr, sd, meta, z


@pytest.mark.parametrize("B", [5, 13])
@pytest.mark.parametrize("name", golden_names("gradrnn_"))
def test_kernels_match_reference_pinned_oracle(name, B):
    """The fixtures' configurations (IC predator-prey with detach_gap cuts, IRIC traffic junction with cars spawning and
    leaving, the predator-prey hard geometry): the kernels against the float64 tanh-RNN oracle replaying every slot
    teacher-forced (tests/rnn_oracle.py; pinned to the unmodified reference by tests/test_oracle_rnn.py), and against
    the float64 backward over the kernel trainer's own records.  B * N is never a multiple of 128: a ragged last tile."""
    from oracle import policy as opolicy
    from rnn_oracle import rnn_oracle
    seed, id0 = 808, 30
    tr, sd, meta, z = fixture_trainer(name, B, seed, id0)
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
    ref, rloss = records_reference(tr)
    for k, r in ref.items():                   # the two float64 yardsticks agree (fp32 records vs float64 rollout)
        assert max_rel_err(r.cpu().numpy(), want[k]) < 1e-5, (name, k)
    label = "%s B=%d %s" % (name, B, events(tr))
    assert_within_bar(tr, got, gloss, oracle, wstat, label + " vs oracle")
    assert_within_bar(tr, got, gloss, ref, rloss, label + " vs float64 records")


@pytest.mark.parametrize("name", golden_names("gradrnn_"))
def test_kernels_match_reference_gradient_arrays(name):
    """One slot with the fixture's seed and env id plays the reference's own batch (same episodes, same actions): the
    kernels' loss sums and gradient against the arrays the unmodified reference's compute_grad produced."""
    meta = load_golden(name)[0]
    tr, sd, meta, z = fixture_trainer(name, 1, meta["seed"], meta["env_id"])
    batch, stat = tr.run_batch(0)
    assert (stat["num_steps"], stat["num_episodes"]) == (meta["num_steps"], meta["num_episodes"])
    got, gloss = grads_of(tr)
    for q in LOSS_KEYS:
        assert np.isclose(gloss[q], meta[q], rtol=2e-4, atol=1e-3), (q, gloss[q], meta[q])
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


# ---------------------------------------------------------------------------------------------------- vs float64

CASES = {
    "pp_ic_detach": (PP, dict(detach_gap=4, max_steps=12, batch_size=30)),
    "tj_iric": (TJ, dict(mean_ratio=0.0)),
    "pp_ic_enemy_entr": ("grad_pp_enemy_ic3net_h128", dict(entr=0.01, normalize_rewards=True)),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("B", [5, 13])
def test_gradient_matches_float64_records(case, B):
    """B * N never a multiple of 128: a ragged last tile."""
    name, over = CASES[case]
    tr = make_trainer(name, B, **over)
    assert tr.grad_kernels and tr.grad_impl == "kernels" and tr.record_mode == "full"
    tr.run_batch(0)
    got, gloss = grads_of(tr)
    ref, rloss = records_reference(tr)
    ev = events(tr)
    if case == "pp_ic_detach":                       # 12-step episodes inside a 30-step quota: restarts and cuts
        assert ev["fresh"] > 0 and ev["cut"] > 0, ev
    assert int(tr._buf["err"].item()) == 0
    assert_within_bar(tr, got, gloss, ref, rloss, "%s B=%d %s" % (case, B, ev))


@pytest.mark.parametrize("name,B", [(PP, 8192), (TJ, 4096)])
def test_full_size_gradient_matches_float64(name, B):
    """81 920 rows (640 tiles), the reference batch boundary."""
    tr = make_trainer(name, B, seed=5, id0=0)
    tr.run_batch(0)
    got, gloss = grads_of(tr)
    ref, rloss = records_reference(tr)
    assert_within_bar(tr, got, gloss, ref, rloss, "%s B=%d" % (name, B))


def _split(np_cols, sms):
    """(j0, j1) of the weight-gradient kernel for one 128-column gate block with the h block as slice 0 (plan_layout)."""
    per_mb = sms // 2
    c0 = 3.0 * (128 + 86) / 3.0
    c1 = 2.0 * (128 + 0.5 * (np_cols - 256) + 22 if np_cols > 256 else 0.5 * np_cols + 22)
    j0 = min(max(int(per_mb * c0 / (c0 + c1) + 0.5), 1), per_mb - 1)
    return j0, per_mb - j0


@pytest.mark.parametrize("case", ["R<16", "R=128k+2", "dgrad-2-tiles", "wgrad-uneven"])
def test_row_counts_around_thresholds(case):
    """Predator-prey hard geometry (10 agents): fewer rows than one block of the tanh kernel, two rows in the last tile,
    dgrad CTAs with two tiles (> SMs tiles), and a tile count neither weight-gradient slice's role count divides."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    N = load_golden(PP)[0]["args"]["nagents"]
    probe = make_trainer(PP, 1)
    e = probe.env.env
    W = 2 * e.vision + 1
    np_cols = (e.obs_positions + 2 * W * W + 1 + 15) // 16 * 16
    j0, j1 = _split(np_cols, sms)
    if case == "R<16":
        B = 1
    elif case == "R=128k+2":
        B = next(b for b in range(13, 10000) if (b * N) % 128 == 2)
    elif case == "dgrad-2-tiles":
        B = next(b for b in range(sms * 128 // N, 100000) if -(-b * N // 128) > sms and (b * N) % 128)
    else:
        B = next(b for b in range(j0 * 128 // N + 1, 100000)
                 if -(-b * N // 128) % j0 and -(-b * N // 128) % j1 and -(-b * N // 128) > j0 + j1)
    tr = make_trainer(PP, B, seed=77, id0=3, batch_size=14, max_steps=10, detach_gap=3)
    R = B * N
    nt = -(-R // 128)
    tr.run_batch(0)
    got, gloss = grads_of(tr)
    ref, rloss = records_reference(tr)
    assert_within_bar(tr, got, gloss, ref, rloss, "%s: B=%d R=%d tiles=%d j0=%d j1=%d SMs=%d" % (case, B, R, nt, j0, j1,
                                                                                               sms))


# ---------------------------------------------------------------------------------------------------- vs autograd

@pytest.mark.parametrize("name,over", [(PP, dict(detach_gap=3, max_steps=8)), (TJ, dict(mean_ratio=0.0))])
def test_gradient_matches_autograd(name, over):
    tk = make_trainer(name, 64, **over)
    ta = make_trainer(name, 64, grad_impl="autograd", **over)
    assert tk.grad_kernels and not ta.grad_kernels
    tk.run_batch(0)
    ta.run_batch(0)
    assert torch.equal(tk._buf["action"], ta._buf["action"])          # one rollout, two backward passes
    gk, sk = grads_of(tk)
    ga, sa = grads_of(ta)
    sums = heads_abs_sums(tk)
    errs = {}
    for k, a in ga.items():
        m = float(a.abs().max())
        if k in sums:
            errs[k] = float(((gk[k] - a).abs() / (TOL * m + 2.0 ** -20 * sums[k])).max()) * TOL
        else:
            errs[k] = float((gk[k] - a).abs().max()) / m
    print("%s %s: %s | losses %s" % (name, over, " ".join("%s %.1e" % kv for kv in errs.items()),
                                     " ".join("%s %.6g/%.6g" % (q, sk[q], sa[q]) for q in LOSS_KEYS)))
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    assert not bad, bad
    for q in LOSS_KEYS:
        assert np.isclose(sk[q], sa[q], rtol=2e-4, atol=1e-3), (q, sk[q], sa[q])


# ---------------------------------------------------------------------------------------------------- determinism

SCHEDULE_T = (1, 2, 5)


def schedule_grads(out_dir):
    """Gradients and losses after cut rollouts of T = 1, 2, 5 steps, as .npy files under out_dir.  Run in this process
    and in a child with IC3_BPTT_OVERLAP=0."""
    tr = make_trainer(PP, 400, seed=13, id0=2)
    for T in SCHEDULE_T:
        tr.rollout(T, 0, quota=0)
        got, s = grads_of(tr)
        for k, v in got.items():
            np.save(os.path.join(out_dir, "T%d_%s.npy" % (T, k)), v.cpu().numpy())
        np.save(os.path.join(out_dir, "T%d_losses.npy" % T), np.array([s[q] for q in LOSS_KEYS]))


def test_repeated_compute_grad_is_bit_identical():
    tr = make_trainer(TJ, 300, mean_ratio=0.0)
    tr.run_batch(0)
    g1, s1 = grads_of(tr)
    g2, s2 = grads_of(tr)
    assert all(torch.equal(g1[k], g2[k]) for k in g1), [k for k in g1 if not torch.equal(g1[k], g2[k])]
    assert s1 == s2


def test_one_stream_schedule_is_bit_identical(tmp_path):
    mine, child = tmp_path / "overlap", tmp_path / "serial"
    mine.mkdir()
    child.mkdir()
    schedule_grads(str(mine))
    env = dict(os.environ, IC3_BPTT_OVERLAP="0")
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_bptt_rnn as m; m.schedule_grads(%r)"
            % (ROOT, TESTS, str(child)))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    files = sorted(os.listdir(mine))
    assert files == sorted(os.listdir(child)) and len(files) > len(SCHEDULE_T)
    for f in files:
        a, b = np.load(mine / f), np.load(child / f)
        assert np.array_equal(a, b), (f, np.abs(a - b).max())


@pytest.mark.parametrize("name,window", [(PP, 4), (TJ, 1)])
def test_windowed_records_are_bit_identical(name, window):
    """Window mode re-runs the index encoder and the SIMT step from the recorded env state: the same h' bit for bit,
    so the same gradient."""
    tf = make_trainer(name, 200, grad_window=window)
    tw = make_trainer(name, 200, grad_window=window, windows=True)
    out = {}
    for tr in (tf, tw):
        tr.run_batch(0)
        out[tr.record_mode] = grads_of(tr)
    assert tf.record_mode == "full" and tw.record_mode == "window"
    assert "rec_c" not in tf._buf and "ck_c" not in tw._buf and "c_abs" not in tw._buf
    (gf, sf), (gw, sw) = out["full"], out["window"]
    assert all(torch.equal(gf[k], gw[k]) for k in gf), [k for k in gf if not torch.equal(gf[k], gw[k])]
    assert sf == sw


def test_records_hold_h_alone():
    """At predator-prey hard, 8192 slots, batch 500 the full records are (T + 1) B N H float32: 24.3 GB, half the LSTM's."""
    tr = make_trainer(PP, 8192, batch_size=500, max_steps=80, mode="mixed")
    T = tr.batch_plan()[0]
    assert T == 579
    nbytes = tr._record_bytes(T)["full"]
    assert nbytes == (T + 1) * 8192 * 10 * 128 * 4
    assert abs(nbytes / 1e9 - 24.3) < 0.05, nbytes


# ---------------------------------------------------------------------------------------------------- refusals

@pytest.mark.parametrize("model,over", [("mlp", {}), ("commnet", dict(commnet=True, recurrent=False, comm_passes=2)),
                                        ("rnn", dict(vision=3)), ("rnn", dict(dim=22, vision=2))])
def test_out_of_scope_configurations_fall_back(model, over):
    """models.MLP, the non-recurrent CommNet (tanh cells with x_tanh / h_from_x), a 7x7 window and an observation
    pattern of more than 512 columns: 'kernels' raises, 'auto' takes autograd."""
    kw = dict(over, model=model)
    if model == "commnet":
        kw["policy_impl"] = "simt"
    with pytest.raises(NotImplementedError):
        make_trainer(PP, 8, **kw)
    tr = make_trainer(PP, 8, grad_impl="auto", **kw)
    assert not tr.grad_kernels and tr.grad_impl == "autograd" and tr.record_mode is None


def test_tanh_cell_with_communication_gets_no_workspace():
    """The library sizes the tanh cell only without communication: comm_mask_zero = 0, hard attention or two passes
    give 0 bytes; the in-scope configuration is sized."""
    from ic3net_b200 import _lib
    lib = _lib.load()
    hd = (C.c_int32 * _lib.MAX_HEADS)(5, 0, 0, 0)
    pol = dict(B=4, N=3, H=128, O=9 * 13, nheads=1, head_dim=hd, hard_attn=0, comm_avg=1, comm_mask_zero=1, env_id0=0, seed=1,
               obs_off=0, obs_vocab=13, obs_ncount=2, cell=_lib.CELL_TANH, passes=1, x_tanh=0, h_from_x=0)
    env = _lib.PPCfg(B=4, N=3, dim=3, vision=1, mode=0, naction=5, env_id0=0, enemy_comm=0, seed=1)

    def nbytes(**kw):
        cfg = _lib.PolicyCfg(**dict(pol, **kw))
        plan = _lib.BpttPlan(cfg=C.pointer(cfg), w=None, pp_env=C.pointer(env), tj_env=None, x_table=None,
                             value_coeff=0.01, entr=0.0, workspace=None)
        return int(lib.ic3_bptt_workspace_bytes(C.byref(plan)))

    for bad in (dict(comm_mask_zero=0), dict(hard_attn=1), dict(passes=2), dict(H=64)):
        assert nbytes(**bad) == 0, bad
    assert nbytes() > 0


# ---------------------------------------------------------------------------------------------------- end to end

@pytest.mark.parametrize("name,mean_ratio", [(PP, 1.0), (PP, 0.0), (TJ, 1.0), (TJ, 0.0)])
def test_train_batch_ic_iric(name, mean_ratio):
    """IC (mean_ratio 1) and IRIC (mean_ratio 0) under grad_impl 'auto': the kernels, finite losses, parameters move."""
    tr = make_trainer(name, 64, grad_impl="auto", mean_ratio=mean_ratio, detach_gap=5)
    assert tr.grad_impl == "kernels" and tr.grad_kernels
    before = tr.optimizer.flat_params.clone()
    for ep in range(2):
        stat = tr.train_batch(ep)
        assert all(math.isfinite(stat[k]) for k in LOSS_KEYS), stat
    assert not torch.equal(before, tr.optimizer.flat_params)
    assert int(tr._buf["err"].item()) == 0
