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

import pytest
import torch

from gpu_harness import (PP, TJ, assert_close, check_ff_records as check_records, ff_chunk_sizes_and_determinism,
                         ff_full_size, ff_gradient_arrays, ff_halted_slots_contribute_nothing, ff_pinned_oracle,
                         ff_trainer as make_trainer, fixture_trainer, rollout_and_grad)
from helpers import golden_names, load_golden

pytestmark = pytest.mark.gpu

SCALAR = "tj_scalar_grad_hard_ic3net_h128"


# ------------------------------------------------------------------------------------------------------- the reference

@pytest.mark.parametrize("B", [5, 13])
@pytest.mark.parametrize("name", golden_names("gradff_"))
def test_kernels_match_reference_pinned_oracle(name, B):
    ff_pinned_oracle(name, B, None)


@pytest.mark.parametrize("name", golden_names("gradff_"))
def test_kernels_match_reference_gradient_arrays(name):
    ff_gradient_arrays(name, None)


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
    """81 920 rows per step at predator-prey hard (8192 slots), 81 920 at traffic-junction hard (4096 slots)."""
    ff_full_size(name, family, over, None)


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
    enc = "affine1.weight" if "affine1.weight" in got else "encoder.weight"
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
    ff_chunk_sizes_and_determinism(family, over, None)


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
    ff_halted_slots_contribute_nothing(name, family, over, None)


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
    with pytest.raises(NotImplementedError, match="kernels_ff"):      # CommNet / IC3Net with the LSTM cell
        make_trainer(PP, 4, "ic3net", recurrent=True, rnn_type="LSTM")
    with pytest.raises(NotImplementedError, match="kernels_ff"):      # recurrent tanh CommNet
        make_trainer(PP, 4, "commnet", recurrent=True, rnn_type="MLP")
    with pytest.raises(NotImplementedError, match="kernels_ff"):      # hid_size 64
        make_trainer(PP, 4, "ic3net", hid_size=64)
    with pytest.raises(NotImplementedError, match="kernels_ff"):      # vision 3: a 7 x 7 window
        make_trainer(PP, 4, "mlp", vision=3)
    # the IC / IRIC baselines (models.RNN, tanh recurrence)
    with pytest.raises(NotImplementedError, match="kernels_ff"):
        fixture_trainer(PP, 4, 1, 0, model="rnn", policy_impl=None, grad_impl="kernels_ff", commnet=False, ic3net=False,
                        hard_attn=False, recurrent=True, rnn_type="MLP", comm_passes=1, share_weights=False,
                        comm_mask_zero=False)
    # the scalar traffic-junction vocabulary, on the non-recurrent CommNet it would cover with the bool one
    with pytest.raises(NotImplementedError):
        fixture_trainer(SCALAR, 4, load_golden(SCALAR)[0]["seed"], 0, policy_impl="simt", grad_window=16,
                        grad_impl="kernels_ff", recurrent=False, rnn_type="MLP", commnet=True, ic3net=False,
                        hard_attn=False, comm_action_one=False)
    # 'auto' still takes autograd for these families; unknown values raise
    tr = make_trainer(PP, 4, "ic3net", grad_impl="auto")
    assert tr.grad_impl == "autograd" and not tr.grad_ff
    for bad in ("kernels_ff_tc", "kernels_ff_tensor"):
        with pytest.raises(ValueError):
            make_trainer(PP, 4, "ic3net", grad_impl=bad)
