"""GPU tests of the hand-written BPTT kernels (csrc/bptt_tc.cu) beyond one 128-row tile: ``Trainer.compute_grad`` on the
kernel path against the float64 reference of tests/bptt_ref.py, which differentiates the same recorded batch.

Covered: the full batch sizes of the BASELINE configs (predator-prey hard at 8192 envs, traffic-junction hard at 4096
envs, 81 920 rows each), a sweep of row counts around the persistent loops' and the weight-gradient role split's
thresholds (derived from the card's SM count), every width of the last block of observation-pattern columns up to the
512-column limit and the fall-back just past it, and the two-stream schedule (repeatability, equality with the
one-stream schedule, the tensor-map cache under two trainers of different geometry).

Bar: per tensor, max error <= 1e-4 of the tensor's largest entry (the bar of tests/test_gpu_grad.py); the encoder weight
also per input column (1e-4 of that column's largest entry plus 1e-6 of the tensor's), so a wrong or lost block of
observation-pattern columns cannot hide behind a large neighbour; the action heads' entries also get 2^-20 of their
sum of |terms| (the comm head's two-logit gradient cancels to a small fraction of that sum, and its fp32 per-row
terms are exact to a few ulps of the sum; a lost row or tile still breaks the bar); loss sums rtol 2e-4, atol 1e-3."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from bptt_ref import LOSS_KEYS, heads_abs_sums, max_rel_err, oracle_grad_sum, tj_record_obs, trainer_reference
from helpers import finish_args, golden_names, load_golden, ns
from oracle import policy as opolicy
from oracle.gen_golden import make_weights

pytestmark = pytest.mark.gpu

TOL = 1e-4                  # per tensor, relative to its largest entry
COL_FLOOR = 1e-6            # encoder columns: floor relative to the whole tensor's largest entry
SUM_FLOOR = 2.0 ** -20      # action heads: floor relative to the sum of |terms| of each entry (16 fp32 ulps)
TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)


def make_trainer(name, B, seed=808, id0=30, grad_impl="kernels", **over):
    """Trainer on the arguments of fixture ``name`` (overridden by ``over``), weights from the fixture's seed."""
    from ic3net_b200 import data
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    meta, z = load_golden(name)
    args = ns(meta["args"], nenvs=B, seed=seed, env_id0=id0, obs_mode="index", use_graph=False, policy_impl="tc",
              record_for_grad=True, grad_impl=grad_impl, **over)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    net = CommNetMLP(args, args.num_inputs)
    sd = make_weights(meta["weights_seed"], args.num_inputs, args.hid_size, args.naction_heads, args.comm_init)
    net.load_state_dict({k: torch.from_numpy(v).float() for k, v in sd.items()})
    return Trainer(args, net, env), sd, z


def kernel_grad(tr):
    """compute_grad of the recorded batch from zeroed gradients: ({name: float64 grad}, loss dict)."""
    tr.optimizer.zero_grad(set_to_none=False)
    s = tr.compute_grad(None)
    grads = {k: p.grad.detach().to(torch.float64).clone() for k, p in tr.policy_net.named_parameters()}
    return grads, s


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


def compare(got, gloss, ref, rloss, label, abs_sums=None):
    """Errors of the kernel gradient against the reference: {tensor: max error / max |ref|} plus
    'encoder.weight[cols]' = worst column error / (1e-4 max |ref col| + 1e-6 max |ref|) * 1e-4 (<= 1e-4 passes), and
    the loss sums' relative errors.  abs_sums (heads_abs_sums): the action heads' entries are allowed 1e-4 of the
    tensor's largest entry plus 2^-20 of their sum of |terms| (reported on the same scale).  Prints; asserts nothing."""
    errs = {}
    for k, r in ref.items():
        if abs_sums is not None and k in abs_sums:
            allowed = TOL * r.abs().max() + SUM_FLOOR * abs_sums[k]
            errs[k] = float(((got[k] - r).abs() / allowed).max()) * TOL
        else:
            errs[k] = max_rel_err(got[k].cpu().numpy(), r.cpu().numpy())
    g, r = got["encoder.weight"], ref["encoder.weight"]
    allowed = TOL * r.abs().amax(0) + COL_FLOOR * r.abs().max()
    errs["encoder.weight[cols]"] = float(((g - r).abs().amax(0) / allowed).max()) * TOL
    unused = [k for k in got if k not in ref]
    for k in unused:                                      # hidd_encoder: not part of the forward, no gradient
        errs[k] = float(got[k].abs().max())
    worst = max(errs, key=errs.get)
    print("%s: worst %s %.2e | %s | losses %s" % (
        label, worst, errs[worst], " ".join("%s %.1e" % (k, v) for k, v in errs.items()),
        " ".join("%s %.6g/%.6g" % (q, gloss[q], rloss[q]) for q in LOSS_KEYS)))
    return errs


def assert_within_bar(tr, got, gloss, ref, rloss, label):
    errs = compare(got, gloss, ref, rloss, label, heads_abs_sums(tr))
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    assert not bad, (label, bad)
    for q in LOSS_KEYS:
        assert np.isclose(gloss[q], rloss[q], rtol=2e-4, atol=1e-3), (label, q, gloss[q], rloss[q])
    return errs


def events(tr):
    """How often the batch exercises the record-dependent branches of the backward."""
    b, args = tr._buf, tr.args
    T = b["T"]
    return dict(halted=int((b["valid"] == 0).sum()), fresh=int(b["s_fresh"][1:].sum()) if T > 1 else 0,
                cut=int((((b["s_tep"] + 1) % args.detach_gap) == 0).sum()) if args.detach_gap <= args.max_steps else 0)


# ---------------------------------------------------------------------------------------------------- the reference

H128 = [n for n in golden_names("grad_") if load_golden(n)[0]["args"]["hid_size"] == 128]


@pytest.mark.parametrize("name", H128)
def test_reference_matches_oracle_and_kernels(name):
    """The float64 reference (fed from the fp32 records) agrees with the oracle's float64 sum over 5 slots, and the
    kernels agree with it."""
    B, seed, id0 = 5, 808, 30
    tr, sd, z = make_trainer(name, B, seed, id0)
    assert tr.grad_kernels
    batch, stat = tr.run_batch(0)
    T, quota = tr.batch_plan()
    got, gloss = kernel_grad(tr)
    ref, rloss = trainer_reference(tr)
    want, wstat, nsteps = oracle_grad_sum(tr.args, z, opolicy.params_to_f64(sd), batch.action.cpu().numpy(),
                                          batch.valid.cpu().numpy(), seed, id0, quota, T)
    assert stat["num_steps"] == nsteps
    worst = 0.0
    for k, r in ref.items():
        err = max_rel_err(r.cpu().numpy(), want[k])
        worst = max(worst, err)
        assert err < 1e-5, (name, k, err)
    for q in LOSS_KEYS:
        assert np.isclose(rloss[q], wstat[q], rtol=2e-4, atol=1e-3), (name, q, rloss[q], wstat[q])
    print(name, "reference vs oracle: worst %.2e" % worst)
    assert_within_bar(tr, got, gloss, ref, rloss, name)


def test_tj_record_obs_equals_the_live_obs_of_the_same_rollout():
    """The traffic-junction observation rebuilt from the recorded state of step t (loc, alive, last_act, route_id;
    Trainer._record_state) equals what ic3_tj_obs writes from the live env state before step t of the same rollout
    (the dense rollout's observation), on every slot and step and across episode resets, for the whole batch and for
    a range of slots.  Every gradient path records the same state, so a trainer without the BPTT kernels is used."""
    from ic3net_b200 import _lib
    name, B, quota = "grad_tj_hard_ic3net_h128", 16, 1 << 30       # no slot halts: every step is recorded
    tr, _, _ = make_trainer(name, B, grad_impl="autograd")
    live, _, _ = make_trainer(name, B, grad_impl="autograd")
    assert not tr.grad_kernels
    T = tr.batch_plan()[0]
    assert T > tr.args.max_steps                                     # the records cross an episode reset
    tr.rollout(T, 0, quota=quota)
    e = live.env.env
    live._alloc(T)
    live._episode_boundary(0)
    live._buf["err"].zero_()
    want = torch.empty(T, B, tr.args.nagents, tr.env.observation_dim, device="cuda")
    for t in range(T):                       # the same rollout one lock-step at a time, observed before each step
        _lib.check(_lib.load().ic3_tj_obs(C.byref(e.cfg), C.byref(e.state), want[t].data_ptr(), _lib.stream()))
        live._enqueue(1, quota=quota)
        assert torch.equal(live._buf["action"][0], tr._buf["action"][t]), t
    for t in range(T):
        assert torch.equal(tj_record_obs(tr, t, 0, B), want[t]), t
        assert torch.equal(tj_record_obs(tr, t, 5, 13), want[t, 5:13]), t
    assert int(tr._buf["err"].item()) == 0 and int(live._buf["err"].item()) == 0


# ---------------------------------------------------------------------------------------------------- full size

@pytest.mark.parametrize("name,B", [("grad_pp_hard_ic3net_h128", 8192), ("grad_tj_hard_ic3net_h128", 4096)])
def test_full_size_gradient_matches_reference(name, B):
    """The BASELINE batch sizes (81 920 rows, 640 tiles: several items per CTA in every persistent loop, ~40 tiles
    per weight-gradient role), reference batch boundary.  The check is shown to be sensitive: the reference without
    the last env slot (in the ragged last tile) fails it."""
    tr, _, _ = make_trainer(name, B, seed=5, id0=0)
    tr.run_batch(0)
    ev = events(tr)
    assert ev["halted"] > 0 or tr.is_tj, ev          # traffic junction never ends an episode early
    assert ev["fresh"] > 0 and ev["cut"] > 0, ev
    got, gloss = kernel_grad(tr)
    ref, rloss = trainer_reference(tr)
    assert_within_bar(tr, got, gloss, ref, rloss, "%s B=%d" % (name, B))
    last, _ = trainer_reference(tr, slots=(B - 1, B))
    dropped = {k: ref[k] - last[k] for k in ref}
    derrs = compare(got, gloss, dropped, rloss, "%s B=%d without the last slot" % (name, B), heads_abs_sums(tr))
    assert any(v > TOL for v in derrs.values()), derrs
    # for the record: heads re-evaluated in float64 on h' instead of read from the fp32 records
    recomputed, closs = trainer_reference(tr, heads_from_records=False)
    compare(got, gloss, recomputed, closs, "%s B=%d, heads re-evaluated" % (name, B))


# ---------------------------------------------------------------------------------------------------- row / tile sweep

def _sweep_batch(case, sms, N, np_cols):
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


@pytest.mark.parametrize("case", ["R<64", "64<R<128", "R=128k+2", "gates-2-items", "dgrad-2-tiles", "wgrad-uneven"])
def test_row_tile_sweep(case):
    """Predator-prey hard geometry (10 agents, dim 20, vision 1) at row counts chosen from the SM count: an empty second
    warpgroup, a partial tile, two rows in the last tile, gates CTAs with two items (> SMs/2 tiles), dgrad CTAs with two
    tiles (> SMs tiles), and a tile count no weight-gradient role subset divides (uneven split, idle roles)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    name = "grad_pp_hard_ic3net_h128"
    N = load_golden(name)[0]["args"]["nagents"]
    probe, _, _ = make_trainer(name, 1)
    B = _sweep_batch(case, sms, N, pattern_columns(probe))
    tr, _, _ = make_trainer(name, B, seed=77, id0=3, batch_size=14, max_steps=10)
    R = B * N
    nt = -(-R // 128)
    j0, j1 = wgrad_split(pattern_columns(tr), sms)
    checks = {"R<64": R < 64, "64<R<128": 64 < R < 128, "R=128k+2": R % 128 == 2, "gates-2-items": 2 * nt > sms,
              "dgrad-2-tiles": nt > sms, "wgrad-uneven": nt % j0 != 0 and nt % j1 != 0}
    assert checks[case], (case, B, R, nt, j0, j1)
    tr.run_batch(0)
    got, gloss = kernel_grad(tr)
    ref, rloss = trainer_reference(tr)
    assert_within_bar(tr, got, gloss, ref, rloss, "%s: B=%d R=%d tiles=%d j0=%d j1=%d SMs=%d" % (case, B, R, nt, j0,
                                                                                                 j1, sms))


# ---------------------------------------------------------------------------------------------------- P-column widths

@pytest.mark.parametrize("fixture,dim,vision,np_cols", [
    ("grad_pp_hard_ic3net_h128", 3, 0, 16),            # last P block NW 16
    ("grad_pp_hard_ic3net_h128", 9, 1, 112),           # NW 112
    ("grad_pp_hard_ic3net_h128", 10, 1, 128),          # NW 128: the paper's medium predator-prey
    ("grad_pp_hard_ic3net_h128", 22, 1, 512),          # 4 x 128: all warpgroups full, the 512-column limit
    ("grad_pp_hard_ic3net_h128", 20, 2, 464),          # NW 80, vision 2 (W^2 = 25, the operand preparation's limit)
    ("grad_pp_hard_ic3net_h128", 21, 2, 496),          # NW 112, vision 2
    ("grad_pp_enemy_ic3net_h128", 10, 1, 128),         # --enemy_comm: the prey is an agent row
])
def test_pattern_column_widths(fixture, dim, vision, np_cols):
    """Every block width of the weight-gradient kernel's observation-pattern slice that the shipped fixtures never
    instantiate, up to np = 512 (192 KB stage ring)."""
    enemy = int(load_golden(fixture)[0]["args"]["enemy_comm"])
    tr, _, _ = make_trainer(fixture, 64, seed=91, id0=7, nfriendly=3, nagents=3 + enemy, dim=dim, vision=vision,
                            batch_size=14, max_steps=10)
    assert tr.grad_kernels and pattern_columns(tr) == np_cols
    tr.run_batch(0)
    got, gloss = kernel_grad(tr)
    ref, rloss = trainer_reference(tr)
    assert_within_bar(tr, got, gloss, ref, rloss, "%s dim %d vision %d np %d" % (fixture, dim, vision, np_cols))


def test_pattern_wider_than_512_columns_falls_back():
    """PP dim 23 / vision 1 needs 560 pattern columns: 'auto' differentiates with autograd, 'kernels' refuses."""
    name = "grad_pp_hard_ic3net_h128"
    tr, _, _ = make_trainer(name, 4, nfriendly=3, nagents=3, dim=23, vision=1, grad_impl="auto")
    assert pattern_columns(tr) == 560
    assert not tr.grad_kernels and tr.grad_impl == "autograd"
    with pytest.raises(NotImplementedError):
        make_trainer(name, 4, nfriendly=3, nagents=3, dim=23, vision=1, grad_impl="kernels")


# ---------------------------------------------------------------------------------------------------- schedule

SCHEDULE_T = (1, 2, 5)         # the parity-indexed buffer sets: one step, both sets once, odd count reusing set 0


def schedule_grads(out_dir):
    """Gradients and losses of compute_grad after cut rollouts of T = 1, 2, 5 steps (one trainer, 400 envs, 32 tiles),
    saved as .npy files under out_dir.  Run in this process and in a child with IC3_BPTT_OVERLAP=0."""
    tr, _, _ = make_trainer("grad_pp_hard_ic3net_h128", 400, seed=13, id0=2)
    for T in SCHEDULE_T:
        tr.rollout(T, 0, quota=0)
        got, s = kernel_grad(tr)
        for k, v in got.items():
            np.save(os.path.join(out_dir, "T%d_%s.npy" % (T, k)), v.cpu().numpy())
        np.save(os.path.join(out_dir, "T%d_losses.npy" % T), np.array([s[q] for q in LOSS_KEYS]))


def test_repeated_compute_grad_is_bit_identical():
    tr, _, _ = make_trainer("grad_pp_hard_ic3net_h128", 400, seed=13, id0=2)
    tr.run_batch(0)
    g1, s1 = kernel_grad(tr)
    g2, s2 = kernel_grad(tr)
    assert all(torch.equal(g1[k], g2[k]) for k in g1), [k for k in g1 if not torch.equal(g1[k], g2[k])]
    assert s1 == s2


def test_one_stream_schedule_is_bit_identical(tmp_path):
    """IC3_BPTT_OVERLAP=0 (read once per process: a child process) keeps the weight-gradient kernel and the look-ahead
    kernels on the caller's stream; the gradients must equal the two-stream schedule's bit for bit."""
    mine, child = tmp_path / "overlap", tmp_path / "serial"
    mine.mkdir()
    child.mkdir()
    schedule_grads(str(mine))
    env = dict(os.environ, IC3_BPTT_OVERLAP="0")
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_bptt_kernels as m; m.schedule_grads(%r)"
            % (ROOT, TESTS, str(child)))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    files = sorted(os.listdir(mine))
    assert files == sorted(os.listdir(child)) and len(files) > len(SCHEDULE_T)
    for f in files:
        a, b = np.load(mine / f), np.load(child / f)
        assert np.array_equal(a, b), (f, np.abs(a - b).max())


def test_trainers_of_different_geometry_alternate():
    """Two trainers with different tile counts and pattern widths share the static tensor-map cache of the weight-
    gradient kernel: A, B, A must leave A's gradient bit-identical (and B's correct)."""
    ta, _, _ = make_trainer("grad_pp_hard_ic3net_h128", 400, seed=13, id0=2)
    tb, _, _ = make_trainer("grad_pp_hard_ic3net_h128", 64, seed=91, id0=7, nfriendly=3, nagents=3, dim=10, vision=1,
                            batch_size=14, max_steps=10)
    assert pattern_columns(ta) != pattern_columns(tb)
    ta.run_batch(0)
    tb.run_batch(0)
    ga1, sa1 = kernel_grad(ta)
    gb, sb = kernel_grad(tb)
    ga2, sa2 = kernel_grad(ta)
    assert all(torch.equal(ga1[k], ga2[k]) for k in ga1) and sa1 == sa2
    ref, rloss = trainer_reference(tb)
    assert_within_bar(tb, gb, sb, ref, rloss, "B after A")
