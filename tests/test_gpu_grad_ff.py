"""The gradient kernels of the non-recurrent tanh policies (ic3_ff_grad_*, grad_impl 'kernels_ff', the backward's
products on the tensor cores in csrc/ff_grad_tc.cu): models.MLP and the CommNet / IC3Net without --recurrent.

Covered:
  - the kernels against the float64 oracle of tests/ff_oracle.py (pinned to the unmodified reference by
    tests/test_oracle_ff.py) replaying every slot teacher-forced, on 5 and 13 slots (ragged tiles), for every gradff_*
    fixture; one slot with a fixture's seed and env id against the reference's stored gradient arrays;
  - the kernels against a float64 backward over the trainer's own records (ff_oracle.records_reference): predator-prey
    hard with 8192 slots and traffic-junction hard with 4096 slots, 1, 2 and 4 passes with and without share_weights,
    comm_mode sum; row counts around every threshold the path uses (128-row dgrad tiles, 256-row heads blocks, the
    256-block row partition of the weight-gradient sums, the persistent grid) with the workspace poisoned (NaN) past
    the rows of each chunk, and 1 .. 32 agents per env; gradients around 1e-6 and 1e2 (both ends of the operand
    scaling);
  - a cross-check against the torch-autograd recompute of the same rollout;
  - chunk sizes K = 1, a K that does not divide T, and K >= T; bit-identical gradients run to run;
  - the pass-state recompute (ic3_policy_ff_states): every h block against ic3_policy_step with that many passes, bit
    for bit, and every S block against the gated mean of the block before it;
  - slots that completed their batch (valid = 0) contribute exactly nothing, whatever their records hold;
  - train_batch end to end for each family on both environments with no device error flag, and the command line;
  - refusals: NotImplementedError outside the kernels' coverage, ValueError for unknown grad_impl values.

Bar (that of tests/test_gpu_bptt_rnn.py): per tensor 1e-4 of its largest entry, the encoder weight also per input column,
the action heads also 2^-20 of their sum of |terms|; loss sums rtol 2e-4."""
import ctypes as C

import numpy as np
import pytest
import torch

from bptt_ref import LOSS_KEYS, max_rel_err, oracle_grad_sum
from ff_oracle import ff_oracle, make_weights, records_reference
from helpers import finish_args, golden_names, load_golden, ns

pytestmark = pytest.mark.gpu

TOL = 1e-4
COL_FLOOR = 1e-6
SUM_FLOOR = 2.0 ** -20
PP, TJ = "grad_pp_hard_ic3net_h128", "grad_tj_hard_ic3net_h128"
FAMILIES = {
    "mlp": dict(model="mlp", commnet=False, hard_attn=False),
    "ic3net": dict(model="commnet", commnet=1, hard_attn=1),
    "commnet": dict(model="commnet", commnet=1, hard_attn=0),
}


def make_trainer(name, B, family, grad_impl="kernels_ff", seed=808, id0=30, weights_seed=77, **over):
    from ic3net_b200 import data, models
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    meta, _ = load_golden(name)
    fam = dict(FAMILIES[family])
    model = fam.pop("model")
    kw = dict(fam, ic3net=False, recurrent=False, rnn_type="MLP", nenvs=B, seed=seed, env_id0=id0, obs_mode="index", use_graph=False,
              policy_impl=None, record_for_grad=True, grad_impl=grad_impl, comm_passes=1, share_weights=False,
              entr=0.01, comm_mask_zero=False)
    kw.update(over)
    args = ns(meta["args"], **kw)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    torch.manual_seed(weights_seed)
    net = {"mlp": models.MLP, "commnet": CommNetMLP}[model](args, args.num_inputs)
    return Trainer(args, net, env)


def grads_of(tr):
    tr.optimizer.zero_grad(set_to_none=False)
    s = tr.compute_grad(None)
    return {k: p.grad.detach().to(torch.float64).clone() for k, p in tr.policy_net.named_parameters()}, s


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


def encoder_name(got):
    return "affine1.weight" if "affine1.weight" in got else "encoder.weight"


def assert_within_bar(got, gloss, ref, rloss, hsum, label):
    """Kernels against a float64 yardstick: per tensor TOL of its largest entry (+ 2^-20 of the heads' sums of |terms|),
    the encoder weight also per input column (TOL of the column's largest entry + 1e-6 of the tensor's)."""
    errs = {}
    for k, r in ref.items():
        m = float(r.abs().max())
        if m == 0.0:
            assert float(got[k].abs().max()) == 0.0, (label, k)
            continue
        allowed = TOL * m + (SUM_FLOOR * hsum[k] if k in hsum else 0.0)
        errs[k] = float(((got[k] - r).abs() / allowed).max()) * TOL
    ek = encoder_name(got)
    g, r = got[ek], ref[ek]
    allowed = TOL * r.abs().amax(0) + COL_FLOOR * r.abs().max()
    errs[ek + "[cols]"] = float(((g - r).abs().amax(0) / allowed).max()) * TOL
    print("%s: %s | losses %s" % (label, " ".join("%s %.1e" % kv for kv in errs.items()),
                                  " ".join("%s %.6g/%.6g" % (q, gloss[q], rloss[q]) for q in LOSS_KEYS)))
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    assert not bad, (label, bad)
    for q in LOSS_KEYS:
        assert np.isclose(gloss[q], rloss[q], rtol=2e-4, atol=1e-3), (label, q, gloss[q], rloss[q])


def check_records(tr, label):
    got, gloss = grads_of(tr)
    ref, rloss, hsum = records_reference(tr)
    assert_within_bar(got, gloss, ref, rloss, hsum, label)
    assert int(tr._buf["err"].item()) == 0
    return got, ref


# ------------------------------------------------------------------------------------------------------- the reference

def fixture_trainer(name, B, seed, id0):
    """Kernel trainer on the arguments and weights of reference fixture ``name`` (tests/golden/gradff_*)."""
    from ic3net_b200 import data, models
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    meta, z = load_golden(name)
    a = meta["args"]
    model = "commnet" if a["commnet"] else "mlp"
    sd = make_weights(meta["weights_seed"], meta["obs_dim"], a["hid_size"], meta["heads"], a.get("comm_init", "uniform"),
                      model, int(a["comm_passes"]), bool(a["share_weights"]))
    args = ns(a, nenvs=B, seed=seed, env_id0=id0, obs_mode="index", use_graph=False, policy_impl=None,
              record_for_grad=True, grad_impl="kernels_ff")
    env = data.init(args.env_name, args)
    finish_args(args, env)
    assert not args.recurrent
    net = (CommNetMLP if model == "commnet" else models.MLP)(args, args.num_inputs)
    net.load_state_dict({k: torch.from_numpy(v).float() for k, v in sd.items()})
    tr = Trainer(args, net, env)
    assert tr.grad_ff
    return tr, sd, meta, z, model


@pytest.mark.parametrize("B", [5, 13])
@pytest.mark.parametrize("name", golden_names("gradff_"))
def test_kernels_match_reference_pinned_oracle(name, B):
    """Every slot replayed teacher-forced by the float64 oracle of the fixture's policy; B * N never a multiple of 64."""
    from oracle import policy as opolicy
    seed, id0 = 808, 30
    tr, sd, meta, z, model = fixture_trainer(name, B, seed, id0)
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
    ref, rloss, hsum = records_reference(tr)
    for k, r in ref.items():                   # the two float64 yardsticks agree (fp32 records vs float64 rollout);
        # the two-logit comm head's gradient cancels to a small part of its terms, whose fp32 log-probs differ
        allowed = 1e-5 * float(oracle[k].abs().max()) + (SUM_FLOOR * hsum[k] if k in hsum else 0.0)
        assert bool(((r - oracle[k]).abs() <= allowed).all()), (name, k, max_rel_err(r.cpu().numpy(), want[k]))
    assert_within_bar(got, gloss, oracle, wstat, hsum, "%s B=%d vs oracle" % (name, B))
    assert_within_bar(got, gloss, ref, rloss, hsum, "%s B=%d vs float64 records" % (name, B))


@pytest.mark.parametrize("name", golden_names("gradff_"))
def test_kernels_match_reference_gradient_arrays(name):
    """One slot with the fixture's seed and env id plays the reference's own batch: the kernels' loss sums and gradient
    against the arrays the unmodified reference's compute_grad produced."""
    meta = load_golden(name)[0]
    tr, sd, meta, z, model = fixture_trainer(name, 1, meta["seed"], meta["env_id"])
    batch, stat = tr.run_batch(0)
    assert (stat["num_steps"], stat["num_episodes"]) == (meta["num_steps"], meta["num_episodes"])
    got, gloss = grads_of(tr)
    for q in LOSS_KEYS:
        assert np.isclose(gloss[q], meta[q], rtol=2e-4, atol=1e-3), (q, gloss[q], meta[q])
    _, _, hsum = records_reference(tr)
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


# ------------------------------------------------------------------------------------------------------- vs float64

@pytest.mark.parametrize("name,family,over", [
    (PP, "mlp", {}),
    (PP, "ic3net", {}),
    (PP, "ic3net", dict(comm_passes=2)),
    (PP, "ic3net", dict(comm_passes=2, share_weights=True)),
    (PP, "commnet", dict(comm_passes=4)),
    (PP, "ic3net", dict(comm_passes=4, share_weights=True)),
    (TJ, "commnet", dict(comm_passes=2, comm_mode="sum")),
    (TJ, "ic3net", dict(comm_passes=4, share_weights=True)),
])
def test_gradient_matches_float64_records(name, family, over):
    tr = make_trainer(name, 13, family, **over)
    tr.run_batch(0)
    check_records(tr, "%s %s %s" % (name, family, over))


@pytest.mark.parametrize("name,family,over", [
    (PP, "ic3net", dict(comm_passes=2)),
    (TJ, "ic3net", dict(comm_passes=2)),
    (PP, "mlp", {}),
    (PP, "ic3net", {}),
    (PP, "commnet", dict(comm_passes=2)),
    (PP, "commnet", dict(comm_passes=2, share_weights=True)),
    (PP, "ic3net", dict(comm_passes=4)),
    (PP, "ic3net", dict(comm_passes=4, share_weights=True)),
    (TJ, "commnet", dict(comm_passes=3, share_weights=True, comm_mode="sum")),
])
def test_full_size_gradient_matches_float64(name, family, over):
    """81 920 rows per step at predator-prey hard (8192 slots), 81 920 at traffic-junction hard (4096 slots).
    tests/test_gpu_ff_tc.py runs it on the tc_ff forward."""
    B = 8192 if name == PP else 4096
    tr = make_trainer(name, B, family, seed=5, id0=0, batch_size=10, **over)
    tr.run_batch(0)
    check_records(tr, "%s B=%d %s %s" % (name, B, family, over))


class _PoisonedWorkspace:
    """Stands in for the trainer module's torch: byte buffers (the gradient workspace) start as 0xFF, a NaN in every
    float lane, so nothing the kernels read past a chunk's rows (or before they write it) goes unnoticed."""

    def __getattr__(self, k):
        return getattr(torch, k)

    @staticmethod
    def empty(*a, **kw):
        t = torch.empty(*a, **kw)
        if kw.get("dtype") == torch.uint8:
            t.fill_(0xFF)
        return t


def poisoned_check(tr, monkeypatch, K, label):
    from ic3net_b200 import trainer as trainer_mod
    tr.FF_CHUNK_STEPS = K
    with monkeypatch.context() as m:
        m.setattr(trainer_mod, "torch", _PoisonedWorkspace())
        check_records(tr, label)
    assert tr.ff_chunk_steps == min(K, tr._buf["T"])


@pytest.mark.parametrize("B", [1, 7, 12, 13, 25, 26, 411, 819, 821, "grid", "grid+1"])
def test_row_counts_around_thresholds(B, monkeypatch):
    """Env counts at predator-prey hard (10 agents: 12 envs = 120 rows per 128-row dgrad tile): one env, one tile, one
    tile + 1 env, fewer rows than the 256 row blocks, 32-row slabs at the block size, the persistent grid (one tile per
    SM: 'grid') and one env past it; 7 envs fill part of one tile, 26 envs (260 rows) give a second heads block of 4
    rows, 411 (4110 rows) 16 or 17 rows per row block.  Each with a chunk size that leaves a ragged last chunk, and with
    one step per chunk."""
    if isinstance(B, str):
        B = 12 * torch.cuda.get_device_properties(0).multi_processor_count + (B == "grid+1")
    tr = make_trainer(PP, B, "ic3net", comm_passes=2, seed=77, id0=3, batch_size=14, max_steps=10)
    tr.run_batch(0)
    T = tr._buf["T"]
    K = next((k for k in range(2, T) if T % k), 1)          # a ragged last chunk: rows past R in the workspace
    poisoned_check(tr, monkeypatch, K, "B=%d R=%d K=%d" % (B, B * tr.args.nagents, K))
    poisoned_check(tr, monkeypatch, 1, "B=%d K=1" % B)


@pytest.mark.parametrize("name,N", [(PP, 1), (PP, 2), (PP, 3), (PP, 11), (PP, 31), (TJ, 32)])
@pytest.mark.parametrize("family,over", [("ic3net", dict(comm_passes=2)), ("commnet", dict(comm_passes=3, comm_mode="sum")),
                                         ("mlp", {})])
def test_agents_per_env(name, N, family, over, monkeypatch):
    """floor(128 / N) envs per dgrad tile, 128 mod N padding rows, 37 envs: a ragged last tile."""
    agents = dict(nagents=N, nfriendly=N) if name == PP else dict(nagents=N)
    tr = make_trainer(name, 37, family, batch_size=6, **agents, **over)
    tr.run_batch(0)
    poisoned_check(tr, monkeypatch, 3, "%s N=%d %s %s" % (name, N, family, over))


@pytest.mark.parametrize("factor", [1e-5, 1e3])
@pytest.mark.parametrize("family,over", [("ic3net", dict(comm_passes=2)), ("mlp", {})])
def test_small_and_large_gradients(factor, family, over):
    """The head weights are scaled after the rollout: d loss / d h_P, and with it every dz, dpre and every gradient but
    the heads', scales by the same factor (|dz| around 1e-6 and 1e2); the records stay as they are."""
    tr = make_trainer(PP, 96, family, **over)
    tr.run_batch(0)
    with torch.no_grad():
        for k, p in tr.policy_net.named_parameters():
            if k.endswith(".weight") and ("heads." in k or "value_head" in k):
                p.mul_(factor)
    got, ref = check_records(tr, "%s %s x%g" % (family, over, factor))
    enc = encoder_name(got)
    scale = float(ref[enc].abs().max())
    assert 1e-9 < scale < 1e6, scale


CASES = [
    (PP, "mlp", {}),
    (PP, "ic3net", {}),
    (PP, "ic3net", dict(comm_passes=2)),
    (PP, "ic3net", dict(comm_passes=4, share_weights=True)),
    (PP, "commnet", dict(comm_passes=2)),
    (TJ, "commnet", dict(comm_passes=3, share_weights=True, comm_mode="sum")),
    (TJ, "ic3net", {}),
    (TJ, "mlp", {}),
]


@pytest.mark.parametrize("name,family,over", CASES)
def test_gradient_matches_autograd(name, family, over):
    B = 96 if name == PP else 48
    ka = make_trainer(name, B, family, **over)
    au = make_trainer(name, B, family, grad_impl="autograd", **over)
    assert ka.grad_ff and not au.grad_ff
    gk, sk = rollout_and_grad(ka)
    assert "ck_h" not in ka._buf and "rec_h" not in ka._buf
    ga, sa = rollout_and_grad(au)
    assert_close(gk, sk, ga, sa)
    assert int(ka._buf["err"].item()) == 0


@pytest.mark.parametrize("family,over", [("mlp", {}), ("ic3net", dict(comm_passes=2))])
def test_chunk_sizes_and_determinism(family, over):
    tr = make_trainer(PP, 40, family, **over)
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


@pytest.mark.parametrize("name,family,over", [(PP, "ic3net", dict(comm_passes=3)), (TJ, "commnet", dict(comm_passes=2)),
                                              (PP, "mlp", {})])
def test_pass_states_equal_policy_step(name, family, over):
    """st_h[p] (p >= 1) equals ic3_policy_step's h_out of the same policy cut to p passes bit for bit (the first p blocks
    of the packed pass weights are that policy's); st_h[0] is tanh(x); st_s[p] is the gated mean of st_h[p]."""
    from ic3net_b200 import _lib
    tr = make_trainer(name, 37, family, **over)
    tr.run_batch(0)
    b, e, net = tr._buf, tr.env.env, tr.policy_net
    lib = _lib.load()
    B, N, H = e.nenvs, tr.args.nagents, tr.args.hid_size
    cfg = net.policy_cfg(B)
    w = net.packed()
    P = max(1, int(cfg.passes))
    t = b["T"] // 2
    ecfg, est = tr._record_state(t)
    x = torch.empty(B * N, H, device=e.device)
    enc = lib.ic3_tj_encoder_index if tr.is_tj else lib.ic3_pp_encoder_index
    s = _lib.stream()
    _lib.check(enc(C.byref(ecfg), C.byref(est), C.byref(cfg), C.byref(w), x.data_ptr(), s))
    hard = bool(tr.args.hard_attn) and bool(tr.args.commnet)
    h_out = torch.empty(B * N, H, device=e.device)
    val, logp = torch.empty(B * N, device=e.device), torch.empty(B * N, sum(tr.args.naction_heads), device=e.device)
    io = _lib.PolicyIO(x=x.data_ptr(), h=x.data_ptr(), comm_action=b["s_comm"][t].data_ptr() if hard else None,
                       alive=b["s_alive"][t].data_ptr(), fresh=b["s_fresh"][t].data_ptr(), h_out=h_out.data_ptr(),
                       value=val.data_ptr(), logp=logp.data_ptr())
    st_h = torch.empty(P + 1, B * N, H, device=e.device)
    st_s = torch.empty(P, B * N, H, device=e.device)
    _lib.check(lib.ic3_policy_ff_states(C.byref(cfg), C.byref(w), C.byref(io), st_h.data_ptr(), st_s.data_ptr(), s))
    for p in range(1, P + 1):
        cut = net.policy_cfg(B)
        cut.passes = p
        _lib.check(lib.ic3_policy_step(C.byref(cut), C.byref(w), C.byref(io), s))
        torch.cuda.synchronize()
        assert torch.equal(st_h[p], h_out), p
    assert torch.allclose(st_h[0], torch.tanh(x), rtol=0, atol=1e-6)
    if cfg.comm_mask_zero:
        return
    fresh = b["s_fresh"][t].bool().unsqueeze(1)
    alive = torch.where(fresh, torch.ones_like(b["s_alive"][t]), b["s_alive"][t]).double()
    n_alive = alive.sum(1, keepdim=True)
    g = alive * (torch.where(fresh, torch.zeros_like(b["s_comm"][t]), b["s_comm"][t]).double() if hard else 1.0)
    den = torch.where(n_alive > 1, n_alive - 1, torch.ones_like(n_alive)) if cfg.comm_avg else torch.ones_like(n_alive)
    gg = g.unsqueeze(-1)
    for p in range(P):
        hv = st_h[p].double().view(B, N, H)
        want = (gg * ((gg * hv).sum(1, keepdim=True) - gg * hv) / den.unsqueeze(-1)).reshape(B * N, H)
        assert torch.allclose(st_s[p].double(), want, rtol=1e-6, atol=1e-6), p


@pytest.mark.parametrize("name,family,over", [(PP, "ic3net", dict(comm_passes=2)), (TJ, "commnet", dict(comm_passes=2))])
def test_halted_slots_contribute_nothing(name, family, over):
    """Slots that complete their batch early leave valid = 0 records.  Every record of those slot-steps is changed -- the
    recorded outputs, rewards, post-step alive mask, the step inputs (fresh, comm_action, alive) and the env state (to
    other in-range positions / routes) -- and the gradient and loss sums stay bit-identical, over chunks of one step
    and of several.  Traffic-junction episodes all run to max_steps, so no slot halts early there: the last three
    lock-steps of half the slots are marked valid = 0 instead (both gradients are taken with that marking), and their
    rewards are left alone: those episodes did not end there, so the rewards reach the returns of earlier real steps."""
    tr = make_trainer(name, 64, family, batch_size=5, **over)
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


@pytest.mark.parametrize("name", [PP, TJ])
@pytest.mark.parametrize("family", ["mlp", "ic3net", "commnet"])
def test_train_batch(name, family):
    tr = make_trainer(name, 64, family, comm_passes=2 if family != "mlp" else 1)
    before = [p.detach().clone() for p in tr.policy_net.parameters()]
    stat = tr.train_batch(0)
    assert int(tr._buf["err"].item()) == 0
    assert stat["num_steps"] > 0 and all(k in stat for k in ("action_loss", "value_loss", "entropy"))
    changed = [not torch.equal(a, p.detach()) for a, p in zip(before, tr.policy_net.parameters())]
    assert any(changed)


def test_command_line(capsys):
    from ic3net_b200 import main as cli
    rc = cli.main(["--env_name", "predator_prey", "--nagents", "3", "--dim", "5", "--max_steps", "20", "--hid_size", "128",
                   "--commnet", "--comm_passes", "2", "--grad_impl", "kernels_ff", "--nenvs", "64", "--num_epochs", "1",
                   "--epoch_size", "1", "--batch_size", "40"])
    out = capsys.readouterr().out
    assert rc == 0 and "Epoch" in out, out[-2000:]


def test_refusals():
    from ic3net_b200 import data, models
    from ic3net_b200.trainer import Trainer
    import test_gpu_tj_scalar as ts
    with pytest.raises(NotImplementedError, match="kernels_ff"):      # CommNet / IC3Net with the LSTM cell
        make_trainer(PP, 4, "ic3net", recurrent=True, rnn_type="LSTM")
    with pytest.raises(NotImplementedError, match="kernels_ff"):      # recurrent tanh CommNet
        make_trainer(PP, 4, "commnet", recurrent=True, rnn_type="MLP")
    with pytest.raises(NotImplementedError, match="kernels_ff"):      # hid_size 64
        make_trainer(PP, 4, "ic3net", hid_size=64)
    with pytest.raises(NotImplementedError, match="kernels_ff"):      # vision 3: a 7 x 7 window
        make_trainer(PP, 4, "mlp", vision=3)
    # the IC / IRIC baselines (models.RNN, tanh recurrence)
    meta, _ = load_golden(PP)
    args = ns(meta["args"], nenvs=4, seed=1, env_id0=0, obs_mode="index", use_graph=False, policy_impl=None,
              record_for_grad=True, grad_impl="kernels_ff", commnet=False, ic3net=False, hard_attn=False,
              recurrent=True, rnn_type="MLP", comm_passes=1, share_weights=False, comm_mask_zero=False)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    with pytest.raises(NotImplementedError, match="kernels_ff"):
        Trainer(args, models.RNN(args, args.num_inputs), env)
    # the scalar traffic-junction vocabulary, on the non-recurrent CommNet it would cover with the bool one
    m, _ = load_golden(ts.GRAD)
    kw = dict(recurrent=False, rnn_type="MLP", commnet=True, ic3net=False, hard_attn=False, comm_action_one=False)
    with pytest.raises(NotImplementedError):
        ts.build(dict(m, args=dict(m["args"], **kw)), 4, "index", "simt", weights=False, record_for_grad=True,
                 grad_window=16, grad_impl="kernels_ff")
    # 'auto' still takes autograd for these families; unknown values raise
    tr = make_trainer(PP, 4, "ic3net", grad_impl="auto")
    assert tr.grad_impl == "autograd" and not tr.grad_ff
    for bad in ("kernels_ff_tc", "kernels_ff_tensor"):
        with pytest.raises(ValueError):
            make_trainer(PP, 4, "ic3net", grad_impl=bad)
