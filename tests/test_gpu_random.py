"""The Random baseline (models.Random, models.py:37-56) on the GPU: ic3_random_policy_step (csrc/random_policy.cu) and
the Trainer / MultiGPUTrainer / CLI path around it.

Covered:
  - every row of a rollout at the full batch sizes of BASELINE c2 (predator-prey hard, 8192 x 10) and c5 (traffic
    junction hard, 4096 x 20) against the float64 oracle of tests/random_oracle.py: value bit-exact, log-probs within
    1e-6 (relative above 1), actions exact wherever the oracle's draw is more than 1e-5 from a CDF edge (fp32 may flip
    a closer one to the neighbouring action, and only to it);
  - explicit draws ("tape") for both streams, the action draws placed just below and above every inner CDF edge of
    every head, for several head layouts;
  - one slot with a reference fixture's seed and env id replays the reference's batch (tests/golden/random_*);
  - the distribution of one full-size step (KS tests) and different draws for different steps and env ids;
  - CUDA-graph replay bit-identical to eager;
  - no parameter moves, the optimizer state stays empty, checkpoints interchange with the reference's Random +
    torch.optim.RMSprop; two ranks reduce to what one process holding both shards computes; the CLI trains."""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from gpu_harness import random_args, random_trainer as make_trainer
from helpers import golden_names, load_golden, ns
import random_oracle as ro

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

def records(tr):
    b = tr._buf
    return {k: b[k].cpu().numpy().copy() for k in ("action", "logp", "value", "reward", "emask", "mini", "ralive",
                                                   "valid")}


def assert_rows(value, logp, act, heads, u, au):
    """GPU outputs of agent rows against the oracle on the same stream-4 words u and action words au."""
    ov, ologp, oact, margin = ro.step(heads, u, au)
    ologp = np.concatenate(ologp, -1)
    assert np.array_equal(value, ov.astype(np.float32))                      # k 2^-24: exact in fp32
    err = np.abs(logp - ologp) / np.maximum(1.0, np.abs(ologp))
    assert err.max() <= 1e-6, err.max()
    clear = margin > 1e-5
    assert np.array_equal(act[clear], oact[clear]), int((act[clear] != oact[clear]).sum())
    assert np.abs(act[~clear] - oact[~clear]).max(initial=0) <= 1
    return int((~clear).sum())


@pytest.mark.parametrize("geometry", ["c2", "c5"])
def test_every_row_against_float64(geometry):
    """Every (step, slot, agent) of a rollout at the full batch size: the oracle draws from the same counters, ticks
    recovered from the env's tick counter and the valid records (a halted slot keeps its tick)."""
    args = random_args(geometry, batch_size=20)
    net, tr = make_trainer(args)
    batch, stat = tr.run_batch(0)
    e = tr.env.env
    B, N, heads = e.nenvs, args.nagents, list(args.naction_heads)
    r = records(tr)
    T = r["valid"].shape[0]
    steps = np.cumsum(r["valid"].astype(np.int64), 0)                          # [T, B] env steps after step t
    tick0 = e.tick.cpu().numpy().astype(np.int64) - steps[-1]
    ids = args.env_id0 + np.arange(B)
    agents = np.broadcast_to(np.arange(N), (B, N))
    near = 0
    for t in range(T):
        ticks = (tick0 + (steps[t - 1] if t else 0))[:, None]
        u = ro.words(args.seed, ids[:, None], ticks, agents).reshape(B * N, -1)
        au = ro.action_words(args.seed, ids[:, None], ticks, agents, len(heads)).reshape(B * N, -1)
        near += assert_rows(r["value"][t], r["logp"][t].reshape(B * N, -1), r["action"][t].reshape(B * N, -1),
                            heads, u, au)
    assert near <= 1e-3 * T * B * N, near


@pytest.mark.parametrize("heads", [(5,), (2,), (4,), (5, 2), (3, 2, 2)])
def test_explicit_draws_at_cdf_edges(heads):
    """Tape for both streams.  Stream-4 words at random, plus rows with all words zero (every logit equal:
    sqrt(-2 ln 2^-24), a uniform head); action draws 256 / 2^24 below and above an inner CDF edge of every head, 0
    and 2^24 - 1."""
    from ic3net_b200 import _lib
    rs = np.random.RandomState(len(heads) * 10 + heads[0])
    B, N = 96, 7
    R = B * N
    u = rs.randint(0, 1 << 24, size=(R, _lib.RANDOM_WORDS)).astype(np.int64)
    u[::5] = 0
    _, ologp, _, _ = ro.step(list(heads), u, np.zeros((R, len(heads)), dtype=np.int64))
    au = np.zeros((R, len(heads)), dtype=np.int64)
    for k, lp in enumerate(ologp):
        cdf = np.cumsum(np.exp(lp), -1)
        edge = rs.randint(0, max(1, lp.shape[1] - 1), size=R)
        side = rs.choice([-256, 256], size=R)
        au[:, k] = np.clip(np.round(cdf[np.arange(R), edge] * 2.0 ** 24).astype(np.int64) + side, 0, (1 << 24) - 1)
        au[::7, k], au[3::7, k] = 0, (1 << 24) - 1
    dev = torch.device("cuda")
    ut = torch.tensor(u.astype(np.uint32).view(np.int32), device=dev)
    # the upper 8 bits of a tape word are ignored
    ut_hi = torch.tensor((u.astype(np.uint32) | np.uint32(0xAB000000)).view(np.int32), device=dev)
    at = torch.tensor(au.astype(np.int32), device=dev)
    A = sum(heads)
    cfg = _lib.PolicyCfg(B=B, N=N, nheads=len(heads), head_dim=(C.c_int32 * _lib.MAX_HEADS)(*heads), env_id0=5,
                         seed=3)
    lib = _lib.load()
    outs = []
    for tape in (ut, ut_hi):
        value, logp = torch.empty(R, device=dev), torch.empty(R, A, device=dev)
        act = torch.full((R, len(heads)), -1, dtype=torch.int32, device=dev)
        io = _lib.PolicyIO(draws=at.data_ptr(), value=value.data_ptr(), logp=logp.data_ptr(), action=act.data_ptr())
        _lib.check(lib.ic3_random_policy_step(C.byref(cfg), C.byref(io), tape.data_ptr(), _lib.stream()))
        torch.cuda.synchronize()
        outs.append((value.cpu().numpy(), logp.cpu().numpy(), act.cpu().numpy()))
    # draws placed 256 / 2^24 from an edge are clear of it; only a second edge closer than that (a head with a
    # probability below 1.5e-5) leaves a draw near one
    assert assert_rows(*outs[0], list(heads), u, au) <= R * len(heads) // 100
    for x, y in zip(*outs):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("name", golden_names("random_"))
def test_one_slot_replays_reference(name):
    """A single slot with the fixture's seed and env id plays the reference's batch: actions, rewards, num_steps,
    num_episodes and success exactly, the loss sums to 2e-4 relative."""
    meta, z = load_golden(name)
    args = ns(meta["args"], nenvs=1, env_id0=meta["env_id"], seed=meta["seed"], obs_mode="index", use_graph=False)
    net, tr = make_trainer(args)
    batch, stat = tr.run_batch(0)
    T = meta["num_steps"]
    assert stat["num_steps"] == T and stat["num_episodes"] == meta["num_episodes"]
    if meta["success"] >= 0:
        assert stat["success"] == meta["success"]
    v = batch.valid.cpu().numpy()[:, 0]
    assert v[:T].all() and not v[T:].any()
    assert np.array_equal(batch.action.cpu().numpy()[:T, 0], z["act"])
    assert np.array_equal(batch.reward.cpu().numpy()[:T, 0], z["reward"].astype(np.float32))
    assert np.array_equal(batch.value.cpu().numpy()[:T, 0], z["value"].astype(np.float32))
    assert np.allclose(batch.logp.cpu().numpy()[:T, 0], z["logp"], rtol=0, atol=2e-6)
    s = tr.compute_grad(batch)
    for q in ("action_loss", "value_loss", "entropy"):
        assert np.isclose(s[q], meta[q], rtol=2e-4, atol=1e-6), (q, s[q], meta[q])


def test_distribution_of_one_full_size_step():
    """One lock-step at c2 (81 920 rows): values against U[0, 1); logit differences of disjoint pairs (z_1 - z_0,
    z_3 - z_2 of the five-way head, what the log-probs keep of the N(0, 1) logits) against N(0, 2).  Neither KS test
    rejects at 1e-3.  The next step and the next env id draw different values."""
    from scipy import stats
    args = random_args("c2")
    net, tr = make_trainer(args)
    tr.rollout(2, 0, quota=0)
    r = records(tr)
    value, logp = r["value"][0].ravel().astype(np.float64), r["logp"][0].reshape(-1, 5).astype(np.float64)
    assert stats.kstest(value, "uniform").pvalue > 1e-3
    d = np.concatenate([logp[:, 1] - logp[:, 0], logp[:, 3] - logp[:, 2]])
    assert stats.kstest(d / np.sqrt(2.0), "norm").pvalue > 1e-3
    v = r["value"].reshape(2, args.nenvs, args.nagents)
    assert (v[0] == v[1]).mean() < 1e-3                          # two steps
    assert (v[0, 0] != v[0, 1]).all()                             # two env ids
    assert value.min() >= 0.0 and value.max() < 1.0


def test_graph_replay_is_bit_identical_to_eager():
    out = []
    for use_graph in (False, True):
        args = random_args("c5", nenvs=256, batch_size=100, use_graph=use_graph)
        net, tr = make_trainer(args)
        recs = []
        for epoch in range(2):                                   # capture, then replay
            tr.run_batch(epoch)
            recs.append(records(tr))
        out.append(recs)
    for a, b in zip(*out):
        for k in a:
            assert np.array_equal(a[k], b[k]), k


def test_train_batch_moves_nothing_and_checkpoints_interchange(tmp_path):
    """train_batch (Trainer and MultiGPUTrainer) leaves the parameter bit-identical, its .grad None and the RMSprop
    state empty, like the reference's optimizer.step() on a parameter without a gradient.  A checkpoint written here
    loads into the reference's Random (one parameter of 3, models.py:43) + torch.optim.RMSprop(alpha 0.97, eps 1e-6),
    and theirs loads here."""
    from ic3net_b200 import main as m
    from ic3net_b200.multi_gpu import MultiGPUTrainer
    args = random_args("c2", nenvs=512, batch_size=100)
    net, tr = make_trainer(args)
    p0 = tr.optimizer.flat_params.clone()
    s = tr.train_batch(0)
    mt = MultiGPUTrainer(args, lambda: tr)
    s2 = mt.train_batch(1)
    for st in (s, s2):
        assert st["num_steps"] >= args.batch_size * args.nenvs and np.isfinite(st["value_loss"])
    assert torch.equal(tr.optimizer.flat_params, p0) and torch.equal(net.parameter.detach(), p0[:3])
    assert net.parameter.grad is None
    assert tr.state_dict()["state"] == {}
    ref_net = torch.nn.Module()                                  # the reference's Random: `parameter`, shape 3
    ref_net.parameter = torch.nn.Parameter(torch.randn(3))
    ref_opt = torch.optim.RMSprop(ref_net.parameters(), lr=args.lrate, alpha=0.97, eps=1e-6)
    ref_opt.step()                                               # trainer.py:254 with no gradient
    assert ref_opt.state_dict()["state"] == {}
    ours = tr.state_dict()
    assert ours["state"] == ref_opt.state_dict()["state"]
    assert {k: v for k, v in ours["param_groups"][0].items() if k in ("lr", "alpha", "eps", "params")} == \
        {k: v for k, v in ref_opt.state_dict()["param_groups"][0].items() if k in ("lr", "alpha", "eps", "params")}
    path = str(tmp_path / "ours.pt")
    log = m.make_log()
    m.update_log(log, dict(s))
    m.save_checkpoint(path, net, log, mt)
    with m._utils_alias():
        d = torch.load(path, weights_only=False)
    ref_net.load_state_dict(d["policy_net"])
    ref_opt.load_state_dict(d["trainer"])
    assert torch.equal(ref_net.parameter.detach(), p0[:3].cpu())
    theirs = str(tmp_path / "theirs.pt")
    with torch.no_grad():
        ref_net.parameter.mul_(2.0)
    with m._utils_alias():
        torch.save(dict(policy_net=ref_net.state_dict(), log=log, trainer=ref_opt.state_dict()), theirs)
    log2 = m.make_log()
    m.load_checkpoint(theirs, net, log2, mt)
    assert torch.equal(net.parameter.detach().cpu(), ref_net.parameter.detach())
    assert len(log2["epoch"].data) == 1 and tr.state_dict()["state"] == {}


def test_cli_trains_random(capsys):
    from ic3net_b200 import main as m
    rc = m.main(["--env_name", "predator_prey", "--nagents", "10", "--dim", "20", "--vision", "1", "--max_steps", "80",
                 "--random", "--num_epochs", "1", "--epoch_size", "1", "--seed", "5"])
    out = capsys.readouterr().out
    assert rc == 0
    lines = out.splitlines()
    assert any(ln.startswith("Epoch 1\tReward") for ln in lines), out[-2000:]
    assert any(ln.startswith("Success: ") for ln in lines), out[-2000:]


def test_cli_refuses_random_recurrent():
    from ic3net_b200 import main as m
    with pytest.raises(ValueError, match="not recurrent"):
        m.main(["--env_name", "predator_prey", "--nagents", "3", "--dim", "5", "--random", "--recurrent",
                "--num_epochs", "1", "--epoch_size", "1", "--nenvs", "4", "--seed", "1"])


def test_two_ranks_reduce_like_one_process():
    """2 ranks (NCCL) x B slots give the statistics and loss sums of one process holding all 2 B slots."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (have %d)" % torch.cuda.device_count())
    B = 64
    with tempfile.TemporaryDirectory() as d:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
               "127.0.0.1", "--master-port", "29733", os.path.join(HERE, "random_nccl_worker.py"), d, str(B)]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
        assert r.returncode == 0, r.stdout.decode()[-4000:]
        ranks = [dict(np.load(os.path.join(d, "rank%d.npz" % k))) for k in range(2)]
    import random_nccl_worker as w
    args, tr = w.build(2 * B, 0)
    stat = tr.train_batch(0)
    for res in ranks:
        assert int(res["num_steps"]) == stat["num_steps"] and int(res["num_episodes"]) == stat["num_episodes"]
        assert int(res["success"]) == stat["success"]
        assert np.allclose(res["reward"], stat["reward"], rtol=1e-6, atol=1e-4)
        assert np.allclose(res["losses"], [stat[k] for k in ("action_loss", "value_loss", "entropy")], rtol=1e-9)
        assert np.array_equal(res["params"], tr.optimizer.flat_params.cpu().numpy())
