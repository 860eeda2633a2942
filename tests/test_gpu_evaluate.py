"""GPU tests of evaluation: greedy actions in the policy kernels (ic3_policy_cfg.greedy), the episode quota of the env
step tail (ic3_rollout_io.episodes) and Trainer.evaluate / MultiGPUTrainer.evaluate.

Greedy rows: the evaluation env is stepped one lock-step at a time at the full sizes of predator-prey hard (8192 slots)
and traffic-junction hard (4096 slots), with max_steps 6 so that every slot starts new episodes.  Each step runs once
sampled and, from the same state, once greedy: value, log-probs and h' must be bit-identical, and the greedy actions must
be the argmax of the float64 step (tests/policy_ref.py) for the LSTM policies, or of the float64 heads on the step's h'
for the tanh policies, except where the top two logits are closer than 1e-5 max(1, |logit|)."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from gpu_harness import (PP, TJ, UPDATE_FF, UPDATE_IC, UPDATES, argmax_check, close, cpu, episode_trainer,
                         head_logits_f64, lstm_direct_step, lstm_outputs, make_lstm_net, same_stat, synthetic,
                         update_trainer)
from helpers import golden_names, load_golden, make_oracle_env
from oracle.rollout import run_episode
from policy_ref import params_f64, step_f64

pytestmark = pytest.mark.gpu

SIMT = dict(policy_impl="simt", grad_impl="autograd")
POLICIES = {"tc": dict(), "simt": SIMT, "tc_ff": dict(UPDATE_FF, model="mlp", commnet=False, hard_attn=False),
            "tc_tanh": dict(UPDATE_IC)}
STATE = ("fresh", "comm", "alive", "t_ep", "h", "c", "halted", "stat_reward", "stat_comm", "stat_success",
         "stat_episodes", "stat_steps")


class F64Weights(object):
    """A policy's kernel weights in float64, for trainer.policy_forward_torch: the float64 step of every tanh variant
    (models.MLP, models.RNN, non-recurrent CommNet / IC3Net)."""

    def __init__(self, net):
        f = lambda v: None if v is None else [t.detach().double() for t in v] if isinstance(v, (list, tuple)) else \
            v.detach().double()
        self._cfg_proto = net._cfg_proto
        self.w = {k: f(v) for k, v in net._kernel_weights().items()}

    def _kernel_weights(self):
        return self.w


def tanh_step_f64(tr, net, obs, h0, comm, alive, fresh):
    """Float64 log-probs [R, sum(heads)] of one step of a tanh policy from its inputs (as Trainer._forward_window)."""
    from ic3net_b200.trainer import policy_forward_torch
    B, N = alive.shape
    f64 = F64Weights(net)
    w = f64.w
    x = obs @ w["enc_w"].t() + w["enc_b"]
    keep = (1 - fresh.double()).repeat_interleave(N).unsqueeze(1)
    fr = fresh.bool().unsqueeze(1)
    al = torch.where(fr, torch.ones_like(alive), alive).double()
    g = al * torch.where(fr, torch.zeros_like(comm), comm).double() if tr.hard else al
    _, _, _, logps = policy_forward_torch(f64, x, h0.double() * keep, torch.zeros_like(x), g, al.sum(1, keepdim=True))
    return torch.cat(logps, 1)


@pytest.mark.parametrize("impl", sorted(POLICIES))
@pytest.mark.parametrize("name,B", [(PP, 8192), (TJ, 4096)])
def test_greedy_every_row(name, B, impl):
    over = dict(POLICIES[impl], record_for_grad=False, grad_impl="auto")
    tr = update_trainer(name, B, False, max_steps=6, eval_nenvs=B, **over)
    assert tr.policy_net.policy_impl == impl
    ev = tr._eval_state()
    e, b = ev["env"], ev["buf"]
    args, net = tr.args, tr.policy_net
    N, heads = args.nagents, list(args.naction_heads)
    R = B * N
    tr._episode_boundary(None, b, e)
    net.packed()
    net.encoder_table(e, force=True)
    lstm = impl in ("tc", "simt")
    P = params_f64(net.state_dict(), 1, device="cuda") if lstm else None
    exempt, nfresh = 0, 0
    for t in range(14):
        snap, saved = e.snapshot(), {k: b[k].clone() for k in STATE if k in b}
        h0, c0 = b["h"].clone(), b["c"].clone()
        comm, alive, fresh = b["comm"].clone(), b["alive"].clone(), b["fresh"].clone()
        nfresh += int(fresh.sum())
        obs = e._get_obs().reshape(R, -1).double()
        tr._enqueue(1, 0, b, e, episodes=3, greedy=False)
        sampled = dict(value=b["value"].clone(), logp=b["logp"].clone(), h=b["h"].clone())
        e.restore(snap)
        for k, v in saved.items():
            b[k].copy_(v)
        tr._enqueue(1, 0, b, e, episodes=3, greedy=True)
        torch.cuda.synchronize()
        for k, v in sampled.items():
            assert torch.equal(b[k], v), "%s %s step %d: greedy %s differs from sampled mode" % (name, impl, t, k)
        act = b["action"][0].reshape(R, -1).cpu().numpy()
        if lstm:
            ref = step_f64(P, obs, h0, c0, comm if tr.hard else None, alive, fresh, nagents=N, passes=1,
                           hard_attn=tr.hard, comm_mode=getattr(args, "comm_mode", "avg"),
                           comm_mask_zero=bool(args.comm_mask_zero))
            logits = head_logits_f64(net, ref[0])
        else:
            logits = tanh_step_f64(tr, net, obs, h0, comm, alive, fresh)
        exempt += argmax_check(logits.cpu().numpy(), act, heads, "%s %s step %d" % (name, impl, t))
    tr.stat_from_vector(tr.stat_vector(b, e).cpu().numpy(), e)      # raises on a device-side flag
    assert nfresh > B
    print("%s %s B=%d: 14 steps x %d rows, near-tie rows exempt: %d" % (name, impl, B, R, exempt))


@pytest.mark.parametrize("heads", [(5, 2), (9, 2), (16, 15)], ids=["fused", "heads16", "heads32"])
def test_greedy_heads_paths(heads):
    """The three head paths of the tensor-core step (fused finish, heads_kernel<16>, heads_kernel<32>): greedy against
    explicit draws from the same inputs, log-probs and value bit-identical, actions the argmax of the float64 heads."""
    N, O, B = 7, 61, 300
    R = B * N
    net, a = make_lstm_net(N, O, heads, wseed=sum(heads))
    inputs = synthetic(B, N, O, seed=len(heads) + sum(heads))
    draws = torch.randint(0, 1 << 24, (R, len(heads)), dtype=torch.int32, device="cuda")
    sampled = lstm_outputs(R, heads)
    assert lstm_direct_step(net, *inputs, sampled, draws=draws) == 0
    proto = net.policy_cfg
    net.policy_cfg = lambda Bn: _greedy(proto(Bn))
    try:
        greedy = lstm_outputs(R, heads)
        assert lstm_direct_step(net, *inputs, greedy, draws=draws) == 0
    finally:
        net.policy_cfg = proto
    for k in ("value", "logp", "h", "c"):
        assert torch.equal(greedy[k], sampled[k]), k
    argmax_check(head_logits_f64(net, greedy["h"]).cpu().numpy(), greedy["action"].cpu().numpy(), heads, str(heads))
    # all logits of a head equal: every row takes index 0 (the lowest tied index, torch.argmax)
    with torch.no_grad():
        for hw, hb in zip(net._kernel_weights()["head_w"], net._kernel_weights()["head_b"]):
            hw.zero_()
            hb.fill_(0.25)
    net.policy_cfg = lambda Bn: _greedy(proto(Bn))
    try:
        tied = lstm_outputs(R, heads)
        assert lstm_direct_step(net, *inputs, tied, draws=draws) == 0
    finally:
        net.policy_cfg = proto
    assert bool((tied["action"] == 0).all()), heads


@pytest.mark.parametrize("impl", sorted(POLICIES))
def test_ties_take_the_lowest_index(impl):
    """Zero action-head weights and equal biases make every logit of a head equal: greedy evaluation picks action 0 in
    every head on every row, on every policy path."""
    tr = update_trainer(PP, 256, False, max_steps=5, eval_nenvs=256, **dict(POLICIES[impl], record_for_grad=False,
                                                                           grad_impl="auto"))
    w = tr.policy_net._kernel_weights()
    with torch.no_grad():
        for hw, hb in zip(w["head_w"], w["head_b"]):
            hw.zero_()
            hb.fill_(-0.5)
    tr.evaluate(1, greedy=True)
    assert bool((tr._eval["buf"]["action"] == 0).all()), impl


@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("name", golden_names("greedy_"))
def test_one_slot_plays_the_reference_greedy_episode(name, impl):
    """The reference's greedy episode (scripts/gen_golden_greedy.py) on the fixture's env ids: actions, rewards, masks,
    success and episode length; values and log-probs to the fp32 bar.  A slot is skipped only where the fixture's top two
    log-probs are close enough for fp32 to flip the argmax."""
    meta, z = load_golden(name)
    ids = meta["env_ids"]
    args, env, net, tr, p = episode_trainer(meta, max(ids) + 1, impl=impl)
    T = args.max_steps
    tr._alloc(T)
    tr._episode_boundary(meta["epoch"])
    tr._buf["err"].zero_()
    net.packed()
    if tr._fused_x():
        tr._encoder_table()
    tr._enqueue(T, 1, greedy=True)                        # get_episode's quota, greedy actions
    stat = tr.collect_stat()
    b = tr._buf
    compared = 0
    for i, env_id in enumerate(ids):
        g = lambda k: z["e%d_%s" % (i, k)]
        L = len(g("act"))
        act = cpu(b["action"])[:L, env_id]
        if not np.array_equal(act, g("act")):
            assert (g("margin")[(act != g("act")).any(-1)] < 1e-5).any(), (name, env_id)
            continue
        compared += 1
        assert np.array_equal(cpu(b["reward"])[:L, env_id], g("reward").astype(np.float32))
        assert np.array_equal(cpu(b["ralive"])[:L, env_id], g("alive"))
        assert np.array_equal(cpu(b["emask"])[:L, env_id], g("emask")[:, 0])
        assert np.array_equal(cpu(b["mini"])[:L, env_id], g("mini"))
        assert int(b["stat_steps"][env_id]) == L and int(b["stat_episodes"][env_id]) == 1
        assert int(b["stat_success"][env_id]) == max(int(g("success")), 0)
        assert close(cpu(b["value"]).reshape(T, -1, args.nagents)[:L, env_id], g("value"))
        lp = np.concatenate([g("logp%d" % k) for k in range(len(meta["heads"]))], -1)
        assert close(cpu(b["logp"])[:L, env_id], lp)
    assert compared >= 1
    assert stat["num_episodes"] == max(ids) + 1


@pytest.mark.parametrize("B", [5, 13])
def test_sampled_evaluation_equals_the_oracle_replay(B):
    """Sampled evaluation of 2 episodes per slot against the float64 oracle on the evaluation env's Philox streams (env
    ids after the training ids), slot by slot: steps, success and reward sums.  A slot with a draw closer than 1e-4 to a
    CDF edge (fp32 may flip it) is skipped."""
    E = 2
    meta, _ = load_golden("ep_pp_hard_ic3net")
    args, env, net, tr, p = episode_trainer(meta, B, impl="tc", eval_nenvs=B, max_steps=30)
    st = tr.evaluate(E)
    ev = tr._eval
    e, b = ev["env"], ev["buf"]
    id0, seed = int(e.cfg.env_id0), int(e.cfg.seed)
    assert id0 == int(env.env.cfg.env_id0) + B
    compared = 0
    for s in range(B):
        orc = make_oracle_env(args)
        t0, steps, succ, rew, safe = 0, 0, 0, np.zeros(args.nagents), True
        for k in range(E):
            ep = run_episode(orc, p, args, seed, id0 + s, tick0=t0, episode=k)
            safe &= bool((ep["margin"] > 1e-4).all())
            t0 += ep["num_steps"]
            steps += ep["num_steps"]
            succ += max(ep["success"], 0)
            rew += ep["reward"].sum(0)
        if not safe:
            continue
        compared += 1
        assert int(b["stat_steps"][s]) == steps and int(b["stat_success"][s]) == succ, s
        assert np.allclose(b["stat_reward"][s].cpu().numpy(), rew, rtol=1e-5, atol=1e-4), s
    assert compared >= B // 2
    assert st["num_episodes"] == E * B


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_sum_like_one_process():
    here = os.path.dirname(os.path.abspath(__file__))
    B = 64
    with tempfile.TemporaryDirectory() as d:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
               "127.0.0.1", "--master-port", "29741", os.path.join(here, "evaluate_nccl_worker.py"), d, str(B)]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
        assert r.returncode == 0, r.stdout.decode()[-4000:]
        ranks = [dict(np.load(os.path.join(d, "rank%d.npz" % k))) for k in range(2)]
    import evaluate_nccl_worker as w
    _, tr = w.build(2 * B, 0)
    stat = tr.evaluate(2)
    for res in ranks:
        assert int(res["num_steps"]) == stat["num_steps"] and int(res["num_episodes"]) == stat["num_episodes"] == 4 * B
        assert int(res["success"]) == stat["success"]
        assert np.allclose(res["reward"], stat["reward"], rtol=1e-6, atol=1e-4)


def _greedy(cfg):
    cfg.greedy = 1
    return cfg


@pytest.mark.parametrize("B", [5, 13, 8192])
@pytest.mark.parametrize("E", [1, 3])
def test_every_slot_plays_its_quota(B, E):
    tr = update_trainer(PP, B, False, max_steps=20, eval_nenvs=B)
    for greedy in (False, True):
        st = tr.evaluate(E, greedy)
        b = tr._eval["buf"]
        assert st["num_episodes"] == E * B
        assert bool((b["stat_episodes"] == E).all()) and bool((b["halted"] == 1).all())
        assert E * B <= st["num_steps"] <= E * B * 20


def test_sampled_evaluation_is_reproducible_and_continues_its_streams():
    a, b = update_trainer(PP, 13, False, eval_nenvs=13), update_trainer(PP, 13, False, eval_nenvs=13)
    s1, s2 = a.evaluate(2), b.evaluate(2)
    same_stat(s1, s2)
    s3 = a.evaluate(2)
    assert s3["num_steps"] != s1["num_steps"] or not np.array_equal(s3["reward"], s1["reward"])


ISOLATION = {"ic3net_full": dict(), "ic3net_windows": dict(windows=True),
             "mlp_ff": dict(UPDATE_FF, model="mlp", commnet=False, hard_attn=False), "ic_tanh": dict(UPDATE_IC),
             "ic3net_graph_update": dict(graph=True), "ic3net_use_graph": dict(use_graph=True)}


@pytest.mark.parametrize("case", sorted(ISOLATION))
def test_evaluation_leaves_training_untouched(case):
    over = dict(ISOLATION[case])
    graph = over.pop("graph", False)
    plain, evald = update_trainer(PP, 1024, graph, **over), update_trainer(PP, 1024, graph, **over)
    for ep in range(UPDATES):
        evald.evaluate(1, greedy=bool(ep % 2))
        same_stat(plain.train_batch(ep), evald.train_batch(ep))
    for x, y in ((plain.optimizer.flat_params, evald.optimizer.flat_params),
                 (plain.optimizer.flat_square_avg, evald.optimizer.flat_square_avg)):
        assert torch.equal(x, y)
    assert torch.equal(plain.env.env.tick, evald.env.env.tick)


def test_evaluation_reads_the_weights_of_replayed_updates():
    """Evaluations between updates, sampled and greedy, eager and replayed (use_graph), of a trainer whose updates are
    replayed (graph_update) equal those of an eager trainer bit for bit: the evaluation env's encoder table follows the
    weights every update leaves."""
    eager, graph = update_trainer(PP, 256, False), update_trainer(PP, 256, True)
    for ep in range(UPDATES + 1):
        for use_graph, greedy in ((False, False), (True, True), (True, False), (False, True)):
            eager.use_graph = graph.use_graph = use_graph
            same_stat(eager.evaluate(1, greedy), graph.evaluate(1, greedy))
        eager.use_graph = graph.use_graph = False
        if ep < UPDATES:
            same_stat(eager.train_batch(ep), graph.train_batch(ep))


@pytest.mark.parametrize("name", [PP, TJ])
def test_graph_replay_equals_eager(name):
    eager, graph = update_trainer(name, 512, False), update_trainer(name, 512, False, use_graph=True)
    for greedy in (False, True, False):
        same_stat(eager.evaluate(2, greedy), graph.evaluate(2, greedy))


def test_traffic_junction_epoch_sets_add_rate_and_recaptures():
    tr = update_trainer(TJ, 256, False, use_graph=True, curr_start=1, curr_end=10, add_rate_min=0.05, add_rate_max=0.2)
    s0 = tr.evaluate(1)
    k0 = tr._graphs["evaluate"][0]
    assert s0["add_rate"] == pytest.approx(0.05 * 256)
    s1 = tr.evaluate(1, epoch=20)
    assert tr._graphs["evaluate"][0] != k0
    assert s1["add_rate"] / s1["num_episodes"] == pytest.approx(tr._eval["env"].add_rate)
    assert tr._eval["env"].add_rate == pytest.approx(0.2, abs=0.011)
    assert tr.env.env.add_rate == pytest.approx(0.05)               # the training env keeps its curriculum
    eager = update_trainer(TJ, 256, False, curr_start=1, curr_end=10, add_rate_min=0.05, add_rate_max=0.2)
    eager.evaluate(1)
    same_stat(s1, eager.evaluate(1, epoch=20))


def test_random_policy_evaluates_sampled_and_refuses_greedy():
    from gpu_harness import random_args, random_trainer
    _, tr = random_trainer(random_args("c2", nenvs=64, max_steps=20))
    st = tr.evaluate(2)
    assert st["num_episodes"] == 2 * 64
    with pytest.raises(ValueError):
        tr.evaluate(1, greedy=True)


def test_multi_gpu_trainer_single_process_equals_trainer():
    from ic3net_b200.multi_gpu import MultiGPUTrainer
    a = update_trainer(PP, 64, False)
    m = MultiGPUTrainer(a.args, lambda: update_trainer(PP, 64, False))
    same_stat(a.evaluate(2, True), m.evaluate(2, True))
