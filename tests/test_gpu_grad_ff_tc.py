"""The tensor-core backward of the non-recurrent tanh policies (grad_impl 'kernels_ff_tc', ic3_ff_grad_plan.impl =
IC3_FF_GRAD_TC, csrc/ff_grad_tc.cu): models.MLP and CommNet / IC3Net without --recurrent.

Covered, at the bar of tests/test_gpu_grad_ff.py (per tensor 1e-4 of its largest entry, the encoder weight also per input
column, the action heads also 2^-20 of their sum of |terms|; loss sums rtol 2e-4), whose checks are re-used here with
every kernels_ff trainer switched to kernels_ff_tc:
  - every gradff_* fixture against the pinned float64 oracle on 5 and 13 slots, and one slot against the reference's
    stored gradient arrays;
  - a float64 backward over the trainer's own records at full size (predator-prey hard with 8192 slots, traffic-junction
    hard with 4096), on forwards from both the SIMT step and the tc_ff step;
  - agreement with kernels_ff on the same records;
  - chunk sizes K = 1, a K not dividing T, K >= T, and bit-identical gradients run to run;
  - slots with valid = 0 contribute exactly nothing;
  - row counts around every tile / grid / row-block threshold of the new kernels with the workspace poisoned (NaN)
    past the rows of each chunk, and 1 .. 32 agents per env;
  - gradients around 1e-6 and 1e2 (both ends of the operand scaling);
  - refusals with NotImplementedError, and the command line."""
import argparse

import pytest
import torch

import test_gpu_grad_ff as gf
from helpers import golden_names

pytestmark = pytest.mark.gpu

PP, TJ = gf.PP, gf.TJ


@pytest.fixture
def tc(monkeypatch):
    """Every kernels_ff trainer tests/test_gpu_grad_ff.py builds (make_trainer, fixture_trainer) runs kernels_ff_tc."""
    orig = gf.ns
    monkeypatch.setattr(gf, "ns", lambda a, **kw: orig(a, **(dict(kw, grad_impl="kernels_ff_tc")
                                                            if kw.get("grad_impl") == "kernels_ff" else kw)))


@pytest.fixture
def tc_fwd(monkeypatch, tc):
    """kernels_ff_tc on the tc_ff forward."""
    orig = gf.ns
    monkeypatch.setattr(gf, "ns", lambda a, **kw: orig(a, **dict(kw, policy_impl="tc_ff")))


def tc_trainer(name, B, family, **over):
    tr = gf.make_trainer(name, B, family, grad_impl="kernels_ff_tc", **over)
    assert tr.grad_ff and tr.grad_impl == "kernels_ff_tc"
    return tr


# ------------------------------------------------------------------------------------------------------- the reference

@pytest.mark.parametrize("name", golden_names("gradff_"))
def test_reference_fixtures(name, tc):
    gf.test_kernels_match_reference_pinned_oracle(name, 5)
    gf.test_kernels_match_reference_pinned_oracle(name, 13)
    gf.test_kernels_match_reference_gradient_arrays(name)


@pytest.mark.parametrize("name", golden_names("gradff_"))
def test_reference_fixtures_tc_ff_forward(name, tc_fwd):
    gf.test_kernels_match_reference_pinned_oracle(name, 13)


# ------------------------------------------------------------------------------------------------------- vs float64

FULL = [
    (PP, "mlp", {}),
    (PP, "ic3net", {}),
    (PP, "commnet", dict(comm_passes=2)),
    (PP, "commnet", dict(comm_passes=2, share_weights=True)),
    (PP, "ic3net", dict(comm_passes=4)),
    (PP, "ic3net", dict(comm_passes=4, share_weights=True)),
    (TJ, "ic3net", dict(comm_passes=2)),
    (TJ, "commnet", dict(comm_passes=3, share_weights=True, comm_mode="sum")),
    (PP, "mlp", dict(policy_impl="tc_ff")),
    (PP, "ic3net", dict(comm_passes=2, policy_impl="tc_ff")),
    (TJ, "ic3net", dict(comm_passes=2, policy_impl="tc_ff")),
]


@pytest.mark.parametrize("name,family,over", FULL)
def test_full_size_gradient_matches_float64(name, family, over):
    """81 920 rows per step (predator-prey hard, 8192 slots; traffic-junction hard, 4096 slots).  The sum-mode case runs
    on the SIMT forward: the tc_ff forward's own error there grows with the number of agents (README)."""
    B = 8192 if name == PP else 4096
    tr = tc_trainer(name, B, family, seed=5, id0=0, batch_size=10, **over)
    tr.run_batch(0)
    gf.check_records(tr, "%s B=%d %s %s" % (name, B, family, over))


@pytest.mark.parametrize("name,family,over", [(PP, "mlp", {}), (PP, "ic3net", dict(comm_passes=2)),
                                              (TJ, "commnet", dict(comm_passes=2, comm_mode="sum")),
                                              (PP, "ic3net", dict(comm_passes=2, policy_impl="tc_ff"))])
def test_agrees_with_simt_kernels(name, family, over):
    """kernels_ff_tc and kernels_ff on the same records (plan.impl switched), within the bar."""
    from ic3net_b200 import _lib
    tr = tc_trainer(name, 96 if name == PP else 48, family, **over)
    tr.run_batch(0)
    g_tc, s_tc = gf.grads_of(tr)
    tr._ff_impl = _lib.FF_GRAD_SIMT
    g_simt, s_simt = gf.grads_of(tr)
    gf.assert_close(g_tc, s_tc, g_simt, s_simt)
    assert s_tc == s_simt                          # the loss sums come from the shared heads kernel
    assert int(tr._buf["err"].item()) == 0


@pytest.mark.parametrize("family,over", [("mlp", {}), ("ic3net", dict(comm_passes=2))])
def test_chunk_sizes_and_determinism(family, over, tc):
    gf.test_chunk_sizes_and_determinism(family, over)


@pytest.mark.parametrize("name,family,over", [(PP, "ic3net", dict(comm_passes=2)), (TJ, "commnet", dict(comm_passes=2))])
def test_halted_slots_contribute_nothing(name, family, over, tc):
    gf.test_halted_slots_contribute_nothing(name, family, over)


# ------------------------------------------------------------------------------------------------------- row counts

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
        gf.check_records(tr, label)
    assert tr.ff_chunk_steps == min(K, tr._buf["T"])


def row_cases():
    """Env counts at predator-prey hard (10 agents: 12 envs = 120 rows per 128-row dgrad tile): one env, one tile, one
    tile + 1 env, fewer rows than the 256 row blocks, 32-row slabs at the block size, the persistent grid (one tile
    per SM) and one env past it."""
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    return [1, 12, 13, 25, 819, 821, 12 * nsm, 12 * nsm + 1]


@pytest.mark.parametrize("which", range(8))
def test_row_counts_around_thresholds(which, monkeypatch):
    B = row_cases()[which]
    tr = tc_trainer(PP, B, "ic3net", comm_passes=2, seed=77, id0=3, batch_size=14, max_steps=10)
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
    tr = tc_trainer(name, 37, family, batch_size=6, **agents, **over)
    tr.run_batch(0)
    poisoned_check(tr, monkeypatch, 3, "%s N=%d %s %s" % (name, N, family, over))


# ------------------------------------------------------------------------------------------------------- scaling

@pytest.mark.parametrize("factor", [1e-5, 1e3])
@pytest.mark.parametrize("family,over", [("ic3net", dict(comm_passes=2)), ("mlp", {})])
def test_small_and_large_gradients(factor, family, over):
    """The head weights are scaled after the rollout: d loss / d h_P, and with it every dz, dpre and every gradient but
    the heads', scales by the same factor (|dz| around 1e-6 and 1e2); the records stay as they are."""
    tr = tc_trainer(PP, 96, family, **over)
    tr.run_batch(0)
    with torch.no_grad():
        for k, p in tr.policy_net.named_parameters():
            if k.endswith(".weight") and ("heads." in k or "value_head" in k):
                p.mul_(factor)
    got, ref = gf.check_records(tr, "%s %s x%g" % (family, over, factor))
    enc = gf.encoder_name(got)
    scale = float(ref[enc].abs().max())
    assert 1e-9 < scale < 1e6, scale


# ------------------------------------------------------------------------------------------------------- refusals

def test_refusals():
    from ic3net_b200 import data, models
    from ic3net_b200.trainer import Trainer
    from helpers import finish_args, load_golden, ns
    import test_gpu_tj_scalar as ts
    with pytest.raises(NotImplementedError, match="kernels_ff_tc"):      # CommNet / IC3Net with the LSTM cell
        tc_trainer(PP, 4, "ic3net", recurrent=True, rnn_type="LSTM")
    with pytest.raises(NotImplementedError, match="kernels_ff_tc"):      # recurrent tanh CommNet
        tc_trainer(PP, 4, "commnet", recurrent=True, rnn_type="MLP")
    with pytest.raises(NotImplementedError, match="kernels_ff_tc"):      # hid_size 64
        tc_trainer(PP, 4, "ic3net", hid_size=64)
    with pytest.raises(NotImplementedError, match="kernels_ff_tc"):      # vision 3: a 7 x 7 window
        tc_trainer(PP, 4, "mlp", vision=3)
    # the IC / IRIC baselines (models.RNN, tanh recurrence)
    meta, _ = load_golden(PP)
    args = ns(meta["args"], nenvs=4, seed=1, env_id0=0, obs_mode="index", use_graph=False, policy_impl=None,
              record_for_grad=True, grad_impl="kernels_ff_tc", commnet=False, ic3net=False, hard_attn=False,
              recurrent=True, rnn_type="MLP", comm_passes=1, share_weights=False, comm_mask_zero=False)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    with pytest.raises(NotImplementedError, match="kernels_ff_tc"):
        Trainer(args, models.RNN(args, args.num_inputs), env)
    # the scalar traffic-junction vocabulary, on the non-recurrent CommNet it would cover with the bool one
    m, _ = load_golden(ts.GRAD)
    kw = dict(recurrent=False, rnn_type="MLP", commnet=True, ic3net=False, hard_attn=False, comm_action_one=False)
    with pytest.raises(NotImplementedError):
        ts.build(dict(m, args=dict(m["args"], **kw)), 4, "index", "simt", weights=False, record_for_grad=True,
                 grad_window=16, grad_impl="kernels_ff_tc")
    # 'auto' still takes autograd for these families; unknown values still raise
    tr = gf.make_trainer(PP, 4, "ic3net", grad_impl="auto")
    assert tr.grad_impl == "autograd" and not tr.grad_ff
    with pytest.raises(ValueError):
        gf.make_trainer(PP, 4, "ic3net", grad_impl="kernels_ff_tensor")


def test_train_batch_and_command_line(capsys):
    tr = tc_trainer(TJ, 64, "ic3net", comm_passes=2)
    before = [p.detach().clone() for p in tr.policy_net.parameters()]
    stat = tr.train_batch(0)
    assert int(tr._buf["err"].item()) == 0 and stat["num_steps"] > 0
    assert any(not torch.equal(a, p.detach()) for a, p in zip(before, tr.policy_net.parameters()))
    from ic3net_b200 import main as cli
    rc = cli.main(["--env_name", "predator_prey", "--nagents", "3", "--dim", "5", "--max_steps", "20", "--hid_size", "128",
                   "--commnet", "--comm_passes", "2", "--grad_impl", "kernels_ff_tc", "--nenvs", "64", "--num_epochs", "1",
                   "--epoch_size", "1", "--batch_size", "40"])
    out = capsys.readouterr().out
    assert rc == 0 and "Epoch" in out, out[-2000:]
