"""Trainer.update, the training update (rollout, returns, advantages, gradient kernels, statistics, RMSprop, weight pack),
run eagerly or, with graph_update, replayed from CUDA graphs.  Each case trains the same seed and initial weights for K
updates eagerly and with graph_update and asserts bit-identical flat parameters, second moments, the last update's
gradients and the stat dicts, and both equal the reference's call sequence (run_batch, zero_grad, compute_grad,
step(grad_div)); plus the device max |c| of ic3_bptt_begin_dev against ic3_bptt_begin, error flags of the rollout and
of the gradient, the refusals, the CLI with --save / --load, and the re-capture rule of the traffic-junction
curriculum."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gpu_harness import UPDATE_FF, UPDATE_IC, UPDATES, same_stat, update_trainer
from helpers import finish_args, load_golden, ns

pytestmark = pytest.mark.gpu

PP, TJ = "grad_pp_hard_ic3net_h128", "grad_tj_hard_ic3net_h128"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def train_both(name, B, epochs=None, **over):
    """(eager trainer, graph trainer) after UPDATES updates each, asserting identical stat dicts along the way."""
    eager, graph = update_trainer(name, B, False, **over), update_trainer(name, B, True, **over)
    for ep in (epochs or range(UPDATES)):
        same_stat(eager.train_batch(ep), graph.train_batch(ep))
    return eager, graph


def assert_same_state(eager, graph):
    oe, og = eager.optimizer, graph.optimizer
    assert torch.equal(oe.flat_params, og.flat_params)
    assert torch.equal(oe.flat_square_avg, og.flat_square_avg)
    assert torch.equal(oe.flat_grads, og.flat_grads)
    assert oe.steps == og.steps == UPDATES


def reference_update(tr, epoch):
    """The reference's Trainer.train_batch (trainer.py:245-256) spelled out on the Trainer's public calls, the divisor
    taken on the host.  models.Random has no gradient: no zero_grad and no step (its parameter keeps .grad None)."""
    from ic3net_b200.utils import merge_stat
    batch, stat = tr.run_batch(epoch)
    if not tr.random_policy:
        tr.optimizer.zero_grad()
    merge_stat(tr.compute_grad(batch), stat)
    if not tr.random_policy:
        tr.optimizer.step(grad_div=stat["num_steps"])
    return stat


CASES = {
    "ic3net_full": dict(),
    "ic3net_windows": dict(windows=True),
    "ic3net_passes2_shared": dict(comm_passes=2, share_weights=True),
    "ic3net_no_cuts": dict(detach_gap=10000),
    "ic_tanh_full": dict(UPDATE_IC),
    "ic_tanh_windows": dict(UPDATE_IC, windows=True),
    "mlp_ff": dict(UPDATE_FF, model="mlp", commnet=False, hard_attn=False),
    "ic3net_ff_passes2": dict(UPDATE_FF, model="commnet", commnet=1, hard_attn=1, comm_passes=2, share_weights=False),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_graph_update_is_bit_identical(case):
    over = dict(CASES[case])
    eager, graph = train_both(PP, 37, **over)                 # 37 x 10 agent rows: a ragged last 128-row tile
    assert_same_state(eager, graph)
    assert graph.update_captures == 1
    if eager.grad_kernels:
        assert eager.record_mode == graph.record_mode == ("window" if over.get("windows") else "full")


@pytest.mark.parametrize("case", sorted(CASES) + ["autograd"])
def test_update_equals_the_reference_sequence(case):
    """UPDATES updates of train_batch, eager and (where it is allowed) with graph_update, equal as many updates of the
    reference's call sequence bit for bit: parameters, second moments, gradients and stat dicts."""
    over = dict(CASES.get(case, dict(grad_impl="autograd")))
    ref = update_trainer(PP, 37, False, **over)
    want = [reference_update(ref, ep) for ep in range(UPDATES)]
    for graph in (False, True) if case in CASES else (False,):
        tr = update_trainer(PP, 37, graph, **over)
        for ep in range(UPDATES):
            same_stat(want[ep], tr.train_batch(ep))
        assert_same_state(ref, tr)


def test_random_update_equals_the_reference_sequence():
    from gpu_harness import random_args, random_trainer as make_random
    ref, tr = (make_random(random_args("c2", nenvs=64, batch_size=100))[1] for _ in range(2))
    p0 = tr.optimizer.flat_params.clone()
    for ep in range(UPDATES):
        same_stat(reference_update(ref, ep), tr.train_batch(ep))
    for t in (ref, tr):
        assert torch.equal(t.optimizer.flat_params, p0)
        assert t.policy_net.parameter.grad is None
        assert t.state_dict()["state"] == {}


def test_use_graph_update_replays_the_rollout_graph():
    """use_graph without graph_update: the update's rollout is replayed from the 'rollout' CUDA graph -- its kernels are
    enqueued only by the warm-up and the capture of the first update -- and every update equals that of a trainer
    without use_graph bit for bit; BPTT kernels and models.Random."""
    from gpu_harness import random_args, random_trainer as make_random
    pairs = [(update_trainer(PP, 37, False), update_trainer(PP, 37, False, use_graph=True)),
             tuple(make_random(random_args("c2", nenvs=64, batch_size=100, use_graph=g))[1] for g in (False, True))]
    for plain, replayed in pairs:
        enqueue, calls = replayed._enqueue, []

        def counted(*args, enqueue=enqueue, calls=calls):
            calls.append(args)
            return enqueue(*args)

        replayed._enqueue = counted
        for ep in range(UPDATES):
            same_stat(plain.train_batch(ep), replayed.train_batch(ep))
        assert len(calls) == 2 and "rollout" in replayed._graphs
        for key in ("action", "logp", "value", "reward"):
            assert torch.equal(plain._buf[key], replayed._buf[key]), key
        for a, b in ((plain.optimizer.flat_params, replayed.optimizer.flat_params),
                     (plain.optimizer.flat_square_avg, replayed.optimizer.flat_square_avg),
                     (plain.optimizer.flat_grads, replayed.optimizer.flat_grads)):
            assert torch.equal(a, b)


BEGIN_CASES = {"full": dict(), "windows": dict(windows=True), "passes3": dict(comm_passes=3), "tanh": dict(UPDATE_IC)}


@pytest.mark.parametrize("case", sorted(BEGIN_CASES))
def test_device_begin_leaves_the_workspace_of_the_host_begin(case):
    """ic3_bptt_begin_dev reduces max |c| on the device; ic3_bptt_begin, which takes it from the host, is its reference
    form.  On one plan, from a zeroed workspace each, the two leave the same bytes: full records (rec_c[1:]), window
    records (the rollout's per-step maxima), three comm passes (the bound grows by P - 1) and the tanh RNN (no c)."""
    from ic3net_b200 import _lib
    tr = update_trainer(PP, 37, False, **BEGIN_CASES[case])
    tr.run_batch(0)
    b, lib, s = tr._buf, _lib.load(), _lib.stream()
    hc = not tr._h_only_records()
    plan = tr._bptt_plan(tr._policy_cfg(), tr.policy_net.packed(), _lib.ptr(tr._encoder_table()) if hc else None)
    ws = torch.zeros(int(lib.ic3_bptt_workspace_bytes(C.byref(plan))), dtype=torch.uint8, device=b["h"].device)
    plan.workspace = ws.data_ptr()
    c = None
    if hc:
        c = b["c_abs"] if tr.record_mode == "window" else b["rec_c"][1:]
    assert tr.record_mode == ("window" if case == "windows" else "full")
    cmax = 0.0 if c is None else float(c.abs().max())
    _lib.check(lib.ic3_bptt_begin(C.byref(plan), cmax, s))
    torch.cuda.synchronize()
    host = ws.clone()
    ws.zero_()
    _lib.check(lib.ic3_bptt_begin_dev(C.byref(plan), _lib.ptr(c), 0 if c is None else c.numel(), s))
    torch.cuda.synchronize()
    assert torch.equal(host, ws)


def test_traffic_junction_curriculum_recaptures_exactly_on_a_step():
    # add_rate moves at epochs 1 and 2 (curr_start 0, curr_end 4, step 0.05): spawn_thr changes, the graph re-captures;
    # the repeated epochs move nothing and must replay the graph they have
    over = dict(normalize_rewards=True, add_rate_min=0.1, add_rate_max=0.3, curr_start=0, curr_end=4)
    eager = update_trainer(TJ, 24, False, **over)
    graph = update_trainer(TJ, 24, True, **over)
    captures, thr = [], []
    for ep in (0, 0, 1, 1, 2):
        same_stat(eager.train_batch(ep), graph.train_batch(ep))
        captures.append(graph.update_captures)
        thr.append(int(graph.env.env.cfg.spawn_thr))
    changes = [i == 0 or thr[i] != thr[i - 1] for i in range(len(thr))]
    assert sum(changes) >= 2
    assert captures == list(np.cumsum(changes))
    for a, b in ((eager.optimizer.flat_params, graph.optimizer.flat_params),
                 (eager.optimizer.flat_square_avg, graph.optimizer.flat_square_avg),
                 (eager.optimizer.flat_grads, graph.optimizer.flat_grads)):
        assert torch.equal(a, b)


def test_packed_weights_stay_current_after_a_replay():
    tr = update_trainer(PP, 8, True)
    tr.train_batch(0)
    net = tr.policy_net
    key = net._packed_key
    net.packed()
    assert net._packed_key == key                            # nothing to re-pack: the replay packed the new weights
    before = {k: v.clone() for k, v in net._bufs.items()}
    net.packed(force=True)
    for k, v in net._bufs.items():
        assert torch.equal(before[k], v), k


def test_fp16_range_flag_raises_after_the_replay():
    """Weights outside the fp16 split range: the same RuntimeError as the eager update, from the statistics vector read
    after the replay (an error word, not a device fault), and the update leaves the parameters as they were."""
    for graph in (False, True):
        tr = update_trainer(PP, 4, graph)
        with torch.no_grad():
            tr.policy_net.f_module.weight_hh.mul_(4000.0)
        before = tr.optimizer.flat_params.clone()
        with pytest.raises(RuntimeError, match="0x200"):
            tr.train_batch(0)
        assert torch.equal(before, tr.optimizer.flat_params)


def test_flag_set_during_the_gradient_raises():
    """A flag the gradient kernels set (here: ERR_FP16_RANGE or-ed into the error word right after them, a plain torch
    op the capture holds) stops the step and raises, eager and replayed; the parameters and second moments stay."""
    from ic3net_b200 import _lib
    for graph in (False, True):
        tr = update_trainer(PP, 4, graph)
        losses = tr._losses_device

        def flagged(*args, tr=tr, losses=losses):
            out = losses(*args)
            tr._buf["err"].bitwise_or_(_lib.ERR_FP16_RANGE)
            return out

        tr._losses_device = flagged
        before = (tr.optimizer.flat_params.clone(), tr.optimizer.flat_square_avg.clone())
        with pytest.raises(RuntimeError, match="0x200"):
            tr.train_batch(0)
        assert torch.equal(before[0], tr.optimizer.flat_params)
        assert torch.equal(before[1], tr.optimizer.flat_square_avg)
        assert tr.optimizer.steps == 0


def test_refusals():
    from ic3net_b200 import data, models
    from ic3net_b200.trainer import Trainer
    with pytest.raises(NotImplementedError, match="autograd"):
        update_trainer(PP, 4, True, grad_impl="autograd")
    with pytest.raises(NotImplementedError, match="forward_grad"):
        update_trainer(PP, 4, True, forward_grad="kernels")
    meta, _ = load_golden(PP)
    args = ns(meta["args"], nenvs=4, seed=1, env_id0=0, obs_mode="index", use_graph=False, recurrent=False,
              random=True, graph_update=True, lrate=1e-3)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    args.recurrent = False
    with pytest.raises(NotImplementedError, match="Random"):
        Trainer(args, models.Random(args, args.num_inputs), env)


def test_cli_epoch_and_save_load_round_trip(tmp_path):
    """One epoch end to end with --graph_update, saved, re-loaded and continued: every checkpoint equals the eager
    run's bit for bit (parameters, RMSprop state, log)."""
    from ic3net_b200 import main as m
    base = ["--env_name", "predator_prey", "--nagents", "3", "--dim", "5", "--vision", "1", "--max_steps", "20",
            "--hid_size", "128", "--ic3net", "--recurrent", "--nenvs", "16", "--num_epochs", "1", "--epoch_size", "2",
            "--batch_size", "30", "--seed", "4", "--detach_gap", "10", "--lrate", "0.001"]
    ck = {}
    for mode, extra in (("eager", []), ("graph", ["--graph_update"])):
        a, b = str(tmp_path / (mode + "_a.pt")), str(tmp_path / (mode + "_b.pt"))
        assert m.main(base + extra + ["--save", a]) == 0
        assert m.main(base + extra + ["--load", a, "--save", b]) == 0
        with m._utils_alias():
            ck[mode] = [torch.load(p, weights_only=False) for p in (a, b)]
    for de, dg in zip(ck["eager"], ck["graph"]):
        for k in de["policy_net"]:
            assert torch.equal(de["policy_net"][k], dg["policy_net"][k]), k
        se, sg = de["trainer"]["state"], dg["trainer"]["state"]
        assert sorted(se) == sorted(sg) and len(se) > 0
        for i in se:
            assert torch.equal(se[i]["square_avg"], sg[i]["square_avg"]) and float(se[i]["step"]) == float(sg[i]["step"])
        for k in ("reward", "action_loss", "value_loss", "num_steps"):
            if k in de["log"]:
                assert np.array_equal(np.asarray(de["log"][k].data), np.asarray(dg["log"][k].data)), k
    assert float(ck["graph"][1]["trainer"]["state"][0]["step"]) == 4.0


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_stay_identical_and_equal_eager(tmp_path):
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "graph_update_nccl_worker.py")
    outs = {}
    for mode in ("eager", "graph"):
        out = tmp_path / mode
        out.mkdir()
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2", "--master-port",
               str(29611 if mode == "eager" else 29612), worker, mode, str(out)]
        subprocess.run(cmd, check=True, cwd=ROOT, timeout=900)
        outs[mode] = [torch.load(str(out / ("rank%d.pt" % r)), weights_only=False) for r in range(2)]
    for mode in outs:
        assert torch.equal(outs[mode][0]["params"], outs[mode][1]["params"])
    for r in range(2):
        for key in ("params", "square_avg", "grads"):
            assert torch.equal(outs["eager"][r][key], outs["graph"][r][key]), key
        assert outs["eager"][r]["stats"] == outs["graph"][r]["stats"]
