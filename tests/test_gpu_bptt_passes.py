"""The BPTT kernels (csrc/bptt_tc.cu) on CommNet / IC3Net with comm_passes > 1 and share_weights.

The backward unit is one (step, comm pass); the states entering passes 1 .. P-1 of a step are re-run from the record
with the rollout's own kernels (ic3_policy_pass_states).  Covered:
  - the re-run states: the last pass equals the record bit for bit, every pass is within 1e-5 of float64;
  - the gradient against the float64 oracle replaying every slot (pinned to the unmodified reference through the
    gradpasses_* fixtures: IC3Net predator-prey with 2 passes and detach_gap, CommNet traffic junction with 3 shared
    passes and comm_mode sum, --enemy_comm with 4 passes) and against the float64 backward over the kernel trainer's
    own records (tests/passes_oracle.py), on ragged last tiles and at the full batch sizes;
  - a cross-check against the torch-autograd windowed recompute of the same rollout;
  - bit-identical gradients run to run, between the two-stream and the one-stream schedule, between full and
    windowed records; the refusal of the tanh-cell families.

Bar against the float64 yardsticks: that of tests/test_gpu_bptt_kernels.py (assert_within_bar).  Against autograd: per
tensor, max |kernels - autograd| <= 1e-4 of the autograd tensor's largest entry, the action heads' entries also 2^-20
of their sum of |terms| (the heads' gradient reads the recorded log-probs, autograd re-evaluates them in fp32); loss
sums rtol 2e-4.  comm_mode 'sum' is cross-checked against autograd on short episodes only: summed messages over
several passes make the recurrence ill-conditioned enough that the two fp32 forwards drift apart over long episodes
(the heads' gradients, which do not depend on the backward recursion at all, then differ too); the float64 anchors
are not affected, since they read the same records as the kernels."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from bptt_ref import heads_abs_sums, max_rel_err, oracle_grad_sum
from helpers import finish_args, golden_names, load_golden, ns
from passes_oracle import make_weights, passes_oracle, records_reference
from policy_ref import params_f64, step_f64
from test_gpu_bptt_kernels import assert_within_bar

TOL = 1e-4
LOSS_KEYS = ("action_loss", "value_loss", "entropy")
TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)


def make_trainer(name, B, passes, share=False, seed=808, id0=30, grad_impl="kernels", windows=False, **over):
    """Trainer on the arguments of fixture ``name`` with ``passes`` comm passes (overridden by ``over``); the module's
    own initialisation under the fixture's weight seed, so two trainers of the same arguments hold the same weights."""
    from ic3net_b200 import data
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    meta, _ = load_golden(name)
    kw = dict(nenvs=B, seed=seed, env_id0=id0, obs_mode="index", use_graph=False, policy_impl="tc", record_for_grad=True,
              grad_impl=grad_impl, comm_passes=passes, share_weights=share)
    kw.update(over)
    args = ns(meta["args"], **kw)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    torch.manual_seed(meta["weights_seed"])
    net = CommNetMLP(args, args.num_inputs)
    tr = Trainer(args, net, env)
    if windows:
        tr.RECORD_BYTES_LIMIT = 0
    return tr


def grads_of(tr):
    """compute_grad of the recorded batch from zeroed gradients: ({name: float64 grad}, loss dict)."""
    tr.optimizer.zero_grad(set_to_none=False)
    s = tr.compute_grad(None)
    return {k: p.grad.detach().to(torch.float64).clone() for k, p in tr.policy_net.named_parameters()}, s


def kernels_vs_autograd(name, B, passes, share=False, **over):
    """The same seeded batch differentiated by the kernels and by autograd: {tensor: error / max |autograd|}."""
    tk = make_trainer(name, B, passes, share, **over)
    ta = make_trainer(name, B, passes, share, grad_impl="autograd", **over)
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
        if m == 0.0:                                   # hidd_encoder: not part of the forward
            assert float(gk[k].abs().max()) == 0.0, k
            continue
        if k in sums:
            errs[k] = float(((gk[k] - a).abs() / (TOL * m + 2.0 ** -20 * sums[k])).max()) * TOL
        else:
            errs[k] = float((gk[k] - a).abs().max()) / m
    label = "%s B=%d passes=%d share=%s %s" % (name, B, passes, share, over)
    print("%s: %s | losses %s" % (label, " ".join("%s %.1e" % kv for kv in errs.items()),
                                  " ".join("%s %.6g/%.6g" % (q, sk[q], sa[q]) for q in LOSS_KEYS)))
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    assert not bad, (label, bad)
    for q in LOSS_KEYS:
        assert np.isclose(sk[q], sa[q], rtol=2e-4, atol=1e-3), (label, q, sk[q], sa[q])
    if share:                                          # one C module: one gradient, added by every pass
        names = [n for n, _ in tk.policy_net.named_parameters()]
        assert not any(n.startswith("C_modules.1") for n in names), names
    return tk


# ---------------------------------------------------------------------------------------------------- the re-run

@pytest.mark.gpu
@pytest.mark.parametrize("name,passes,share", [("grad_pp_hard_ic3net_h128", 3, False),
                                               ("grad_tj_hard_ic3net_h128", 2, True)])
def test_pass_states_rerun(name, passes, share):
    """ic3_policy_pass_states from the record of step t: the last pass equals the recorded (h_t, c_t) bit for bit, every
    pass is within 1e-5 of the float64 step with that many passes."""
    from ic3net_b200 import _lib
    tr = make_trainer(name, 96, passes, share, max_steps=5)
    T = 9
    tr.rollout(T, 0)
    tr.collect_stat()
    b, e, net, args = tr._buf, tr.env.env, tr.policy_net, tr.args
    B, N, H = e.nenvs, args.nagents, args.hid_size
    R = B * N
    assert int(b["s_fresh"][1:].sum()) > 0                       # episode starts inside the rollout
    lib = _lib.load()
    cfg = net.policy_cfg(B)
    cfg.seed, cfg.env_id0 = e.cfg.seed, e.cfg.env_id0
    w = net.packed()
    table = tr._encoder_table()
    ws, _ = net.workspace(B)
    hard = bool(args.hard_attn) and bool(args.commnet)
    P = params_f64(net.state_dict(), passes, device="cuda")
    kw = dict(nagents=N, hard_attn=hard, comm_mode=getattr(args, "comm_mode", "avg"),
              comm_mask_zero=bool(args.comm_mask_zero))
    hp = torch.empty(passes, R, H, device="cuda")
    cp = torch.empty(passes, R, H, device="cuda")
    worst = 0.0
    for t in range(T):
        ecfg, est = tr._record_state(t)
        io = _lib.PolicyIO(x=None, h=b["rec_h"][t].data_ptr(), c=b["rec_c"][t].data_ptr(),
                           comm_action=b["s_comm"][t].data_ptr() if hard else None, alive=b["s_alive"][t].data_ptr(),
                           fresh=b["s_fresh"][t].data_ptr(), workspace=_lib.ptr(ws), err=b["err"].data_ptr(),
                           x_table=table.data_ptr(), **_lib.env_source(ecfg, est))
        _lib.check(lib.ic3_policy_pass_states(C.byref(cfg), C.byref(w), C.byref(io), passes, hp.data_ptr(),
                                              cp.data_ptr(), _lib.stream()))
        torch.cuda.synchronize()
        assert torch.equal(hp[-1], b["rec_h"][t + 1]) and torch.equal(cp[-1], b["rec_c"][t + 1]), t
        if tr.is_tj:
            from bptt_ref import tj_record_obs
            obs = tj_record_obs(tr, t, 0, B).reshape(R, -1).double()
        else:
            idx, val = tr._pp_sparse_obs(b["s_loc"][t])
            obs = (idx, val.double())
        for p in range(passes):
            h2, c2, _, _ = step_f64(P, obs, b["rec_h"][t], b["rec_c"][t], b["s_comm"][t], b["s_alive"][t],
                                    b["s_fresh"][t], passes=p + 1, **kw)
            for got, ref in ((hp[p], h2), (cp[p], c2)):
                err = float(((got.double() - ref).abs() / ref.abs().clamp(min=1.0)).max())
                worst = max(worst, err)
                assert err <= 1e-5, (t, p, err)
    assert int(b["err"].item()) == 0
    print("%s passes %d: worst re-run error %.2e over %d steps" % (name, passes, worst, T))


# ---------------------------------------------------------------------------------------------------- vs autograd

@pytest.mark.gpu
@pytest.mark.parametrize("name,passes,share,over", [
    ("grad_pp_hard_ic3net_h128", 2, False, dict(detach_gap=3, max_steps=8)),
    ("grad_tj_hard_ic3net_h128", 3, True, dict(comm_mode="sum", hard_attn=False, max_steps=4)),
    ("grad_pp_enemy_ic3net_h128", 4, False, {}),
    ("grad_pp_hard_ic3net_h128", 3, True, dict(max_steps=6)),
])
def test_gradient_matches_autograd(name, passes, share, over):
    tk = kernels_vs_autograd(name, 64, passes, share, **over)
    b, args = tk._buf, tk.args
    assert int(b["s_fresh"][1:].sum()) > 0
    if args.detach_gap <= args.max_steps:
        assert int((((b["s_tep"] + 1) % args.detach_gap) == 0).sum()) > 0


# ---------------------------------------------------------------------------------------------------- float64 anchors

@pytest.mark.gpu
@pytest.mark.parametrize("B", [5, 13])
@pytest.mark.parametrize("name", golden_names("gradpasses_"))
def test_kernels_match_reference_pinned_oracle(name, B):
    """The fixtures' configurations (IC3Net predator-prey hard geometry with 2 passes and detach_gap, CommNet traffic
    junction with 3 passes of one shared C module and comm_mode sum, --enemy_comm with 4 passes): the kernels against
    the float64 oracle replaying every slot teacher-forced (tests/passes_oracle.py; pinned to the unmodified reference
    by tests/test_oracle_passes.py), and against the float64 backward over the kernel trainer's own records.  B * N is
    never a multiple of 128: a ragged last tile (13 slots of 10 agents: 130 rows, two rows in the second tile)."""
    from ic3net_b200 import data
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    from oracle import policy as opolicy
    meta, z = load_golden(name)
    seed, id0 = 808, 30
    args = ns(meta["args"], nenvs=B, seed=seed, env_id0=id0, obs_mode="index", use_graph=False, policy_impl="tc",
              record_for_grad=True, grad_impl="kernels")
    passes, share = int(args.comm_passes), bool(args.share_weights)
    assert (B * args.nagents) % 128 != 0
    env = data.init(args.env_name, args)
    finish_args(args, env)
    net = CommNetMLP(args, args.num_inputs)
    sd = make_weights(meta["weights_seed"], args.num_inputs, args.hid_size, args.naction_heads, args.comm_init, passes,
                      share)
    net.load_state_dict({k: torch.from_numpy(v).float() for k, v in sd.items()})
    tr = Trainer(args, net, env)
    assert tr.grad_kernels
    batch, stat = tr.run_batch(0)
    T, quota = tr.batch_plan()
    got, gloss = grads_of(tr)
    with passes_oracle(passes, share):
        want, wstat, nsteps = oracle_grad_sum(args, z, opolicy.params_to_f64(sd), batch.action.cpu().numpy(),
                                              batch.valid.cpu().numpy(), seed, id0, quota, T)
    assert stat["num_steps"] == nsteps
    oracle = {k: torch.as_tensor(want[k], device="cuda") for k in got if want.get(k) is not None and np.any(want[k])}
    ref, rloss = records_reference(tr)
    for k, r in ref.items():                   # the two float64 yardsticks agree (fp32 records vs float64 rollout)
        assert max_rel_err(r.cpu().numpy(), want[k]) < 1e-5, (name, k)
    label = "%s B=%d" % (name, B)
    assert_within_bar(tr, got, gloss, oracle, wstat, label + " vs oracle")
    assert_within_bar(tr, got, gloss, ref, rloss, label + " vs float64 records")


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,passes,share", [("grad_pp_hard_ic3net_h128", 8192, 2, False),
                                                 ("grad_tj_hard_ic3net_h128", 4096, 3, True)])
def test_full_size_gradient_matches_float64(name, B, passes, share):
    """81 920 rows (640 tiles, ragged weight-gradient role subsets), the reference batch boundary, against the float64
    backward over the kernel trainer's own records (every comm pass re-run in float64); worst error per tensor printed."""
    tr = make_trainer(name, B, passes, share, seed=5, id0=0)
    tr.run_batch(0)
    got, gloss = grads_of(tr)
    ref, rloss = records_reference(tr)
    assert_within_bar(tr, got, gloss, ref, rloss, "%s B=%d passes=%d share=%s" % (name, B, passes, share))


# ---------------------------------------------------------------------------------------------------- determinism

SCHEDULE_T = (1, 2, 5)


def schedule_grads(out_dir):
    """Gradients and losses after cut rollouts of T = 1, 2, 5 steps with 3 comm passes (odd unit counts), as .npy files
    under out_dir.  Run in this process and in a child with IC3_BPTT_OVERLAP=0."""
    tr = make_trainer("grad_pp_hard_ic3net_h128", 400, 3, seed=13, id0=2)
    for T in SCHEDULE_T:
        tr.rollout(T, 0, quota=0)
        got, s = grads_of(tr)
        for k, v in got.items():
            np.save(os.path.join(out_dir, "T%d_%s.npy" % (T, k)), v.cpu().numpy())
        np.save(os.path.join(out_dir, "T%d_losses.npy" % T), np.array([s[q] for q in LOSS_KEYS]))


@pytest.mark.gpu
def test_repeated_compute_grad_is_bit_identical():
    tr = make_trainer("grad_tj_hard_ic3net_h128", 300, 2, True)
    tr.run_batch(0)
    g1, s1 = grads_of(tr)
    g2, s2 = grads_of(tr)
    assert all(torch.equal(g1[k], g2[k]) for k in g1), [k for k in g1 if not torch.equal(g1[k], g2[k])]
    assert s1 == s2


@pytest.mark.gpu
def test_one_stream_schedule_is_bit_identical(tmp_path):
    mine, child = tmp_path / "overlap", tmp_path / "serial"
    mine.mkdir()
    child.mkdir()
    schedule_grads(str(mine))
    env = dict(os.environ, IC3_BPTT_OVERLAP="0")
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_bptt_passes as m; m.schedule_grads(%r)"
            % (ROOT, TESTS, str(child)))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    files = sorted(os.listdir(mine))
    assert files == sorted(os.listdir(child)) and len(files) > len(SCHEDULE_T)
    for f in files:
        a, b = np.load(mine / f), np.load(child / f)
        assert np.array_equal(a, b), (f, np.abs(a - b).max())


@pytest.mark.gpu
@pytest.mark.parametrize("name,passes,share", [("grad_pp_hard_ic3net_h128", 2, False),
                                               ("grad_tj_hard_ic3net_h128", 4, True)])
def test_windowed_records_are_bit_identical(name, passes, share):
    tf = make_trainer(name, 200, passes, share, grad_window=4)
    tw = make_trainer(name, 200, passes, share, grad_window=4, windows=True)
    out = {}
    for tr in (tf, tw):
        tr.run_batch(0)
        out[tr.record_mode] = grads_of(tr)
    assert tf.record_mode == "full" and tw.record_mode == "window"
    (gf, sf), (gw, sw) = out["full"], out["window"]
    assert all(torch.equal(gf[k], gw[k]) for k in gf), [k for k in gf if not torch.equal(gf[k], gw[k])]
    assert sf == sw


# ---------------------------------------------------------------------------------------------------- refusals

def test_tanh_cells_get_no_workspace(built_lib):
    """ic3_bptt_workspace_bytes checks the policy variant itself: 0 for the tanh cell, x_tanh, h_from_x and more comm
    passes than the policy kernels run; the LSTM cell with 1 .. 4 passes is sized (more with more passes).  Host-side
    checks only, so this runs without a GPU."""
    from ic3net_b200 import _lib
    lib = _lib.load()
    hd = (C.c_int32 * _lib.MAX_HEADS)(5, 2, 0, 0)
    pol = dict(B=4, N=3, H=128, O=99, nheads=2, head_dim=hd, hard_attn=1, comm_avg=1, comm_mask_zero=0, env_id0=0, seed=1,
               obs_off=0, obs_vocab=13, obs_ncount=2, cell=_lib.CELL_LSTM, passes=1, x_tanh=0, h_from_x=0)
    env = _lib.PPCfg(B=4, N=3, dim=3, vision=1, mode=0, naction=5, env_id0=0, enemy_comm=0, seed=1)

    def nbytes(**kw):
        cfg = _lib.PolicyCfg(**dict(pol, **kw))
        plan = _lib.BpttPlan(cfg=C.pointer(cfg), w=None, pp_env=C.pointer(env), tj_env=None, x_table=None,
                             value_coeff=0.01, entr=0.0, workspace=None)
        return int(lib.ic3_bptt_workspace_bytes(C.byref(plan)))

    for bad in (dict(cell=_lib.CELL_TANH), dict(x_tanh=1), dict(h_from_x=1), dict(cell=_lib.CELL_TANH, x_tanh=1, h_from_x=1),
                dict(passes=_lib.MAX_PASSES + 1)):
        assert nbytes(**bad) == 0, bad
    if not torch.cuda.is_available():
        return                                          # sizing the supported ones asks the device for its SM count
    sizes = [nbytes(passes=p) for p in range(1, _lib.MAX_PASSES + 1)]
    assert sizes[0] > 0 and all(a < b for a, b in zip(sizes, sizes[1:])), sizes


@pytest.mark.gpu
def test_tanh_cell_kernels_are_refused():
    """The non-recurrent CommNet (tanh cell) with two passes at the Trainer level: 'kernels' raises, 'auto' takes
    autograd.  The tanh cell runs on the SIMT policy kernel (the tensor-core path refuses it), so the Trainer refuses
    through the missing fused encoder before the cell check; the library's own refusal of the tanh cells is
    test_tanh_cells_get_no_workspace."""
    tanh = dict(recurrent=False, rnn_type="MLP", policy_impl="simt")
    with pytest.raises(NotImplementedError):
        make_trainer("grad_pp_hard_ic3net_h128", 8, 2, **tanh)
    tr = make_trainer("grad_pp_hard_ic3net_h128", 8, 2, grad_impl="auto", **tanh)
    assert tr.policy_net.is_variant and not tr.policy_net.tc_capable
    assert not tr.grad_kernels and tr.grad_impl == "autograd"
