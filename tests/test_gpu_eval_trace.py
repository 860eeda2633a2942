"""GPU tests of the evaluation recorder: Trainer.evaluate_trace (csrc/eval_trace.cu, ic3_trace_step and
ic3_comm_map_step; the out_loc / out_success hooks of the env step kernels) against the float64 oracle slot by slot, its
comm map against a numpy aggregation of its trace, and recording changing nothing that evaluate computes."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from gpu_harness import (PP, TJ, UPDATE_IC, close, episode_trainer, random_args, random_trainer, same_stat,
                         update_trainer)
from helpers import load_golden, make_oracle_env, tj_tables
from greedy_oracle import greedy
from oracle import policy as opolicy
from oracle.rollout import run_episode

pytestmark = pytest.mark.gpu

ORACLE_CASES = {"pp_mixed": ("ep_pp_hard_ic3net", 30), "pp_enemy": ("ep_pp_enemy_ic3net", 20),
                "tj_hard": ("ep_tj_hard_ic3net", 30)}


def _watch(orc, is_tj):
    """Wrap the oracle env so that it logs positions (and, traffic junction, alive mask and routes) at every reset,
    before every step and after every step."""
    log = dict(reset=[], before=[], after=[])
    reset, step = orc.reset, orc.step

    def state():
        if is_tj:
            return dict(loc=orc.car_loc.copy(), alive=orc.alive.copy(), route=orc.route_id.copy())
        return dict(loc=np.concatenate([orc.predator_loc, orc.prey_loc]).copy())

    def r(*a, **k):
        out = reset(*a, **k)
        log["reset"].append(state())
        return out

    def s(*a, **k):
        log["before"].append(state())
        out = step(*a, **k)
        log["after"].append(state())
        return out
    orc.reset, orc.step = r, s
    return log


def _trace_vs_oracle(args, z, p, trace, seed, E, sampled, label):
    """Compare every recorded slot of a trace with the oracle's replay of that slot, the oracle's env following the
    recorded actions.  The oracle's own action (inverse CDF on the same draw, or argmax) must equal the recorded one
    wherever its draw is at least 1e-4 from a CDF edge (sampled) or its top two log-probs at least 1e-5 apart (greedy);
    returns how many slots had no such near tie."""
    is_tj = args.env_name == "traffic_junction"
    heads = list(args.naction_heads)
    hard = bool(args.hard_attn) and bool(args.commnet)
    comm_col = sum(heads) - heads[-1] + 1
    compared = 0
    for j, env_id in enumerate(trace.env_id):
        orc = make_oracle_env(args, tj_tables(z) if is_tj else None)
        log = _watch(orc, is_tj)
        t0, eps, safe = 0, [], True
        for k in range(E):
            ep = run_episode(orc, p, args, seed, int(env_id), tick0=t0, episode=k,
                             forced_actions=trace.action[t0:t0 + args.max_steps, j].astype(np.int64))
            L = ep["num_steps"]
            own = np.array([opolicy.sample_actions(np.split(ep["logp"][t], np.cumsum(heads)[:-1], -1),
                                                   opolicy.action_draws(seed, int(env_id), t0 + t, args.nagents,
                                                                        len(heads)))[0] for t in range(L)])
            far = ep["margin"] > (1e-4 if sampled else 1e-5)
            assert np.array_equal(own[far], trace.action[t0:t0 + L, j][far]), (label, j, k)
            safe &= bool(far.all())
            eps.append((t0, ep))
            t0 += L
        compared += int(safe)
        at = 0
        for k, (s0, ep) in enumerate(eps):
            L = ep["num_steps"]
            sl = slice(s0, s0 + L)
            lab = "%s slot %d episode %d" % (label, j, k)
            assert trace.valid[sl, j].all(), lab
            assert np.array_equal(trace.action[sl, j], ep["act"]), lab
            assert np.array_equal(trace.t_ep[sl, j], np.arange(L)), lab
            done = np.zeros(L, np.uint8)
            done[-1] = 1
            assert np.array_equal(trace.done[sl, j], done), lab
            succ = np.zeros(L, np.uint8)
            succ[-1] = 1 if ep["success"] > 0 else 0
            assert np.array_equal(trace.success[sl, j], succ), lab
            assert np.array_equal(trace.reward[sl, j], ep["reward"].astype(np.float32)), lab
            assert close(trace.value[sl, j], ep["value"]), lab
            nxt = np.stack([log["after"][at + i]["loc"] for i in range(L)])
            assert np.array_equal(trace.loc_next[sl, j], nxt), lab
            assert np.array_equal(trace.loc[s0, j], log["reset"][k]["loc"]), lab
            assert np.array_equal(trace.loc[s0 + 1:s0 + L, j], trace.loc_next[s0:s0 + L - 1, j]), lab
            if is_tj:
                before = np.stack([log["before"][at + i]["alive"] for i in range(L)])
                assert np.array_equal(trace.alive[sl, j], before), lab
                routes = np.stack([log["before"][at + i]["route"] for i in range(L)])
                assert np.array_equal(trace.route_id[sl, j], routes), lab
            else:
                assert (trace.alive[sl, j] == 1).all(), lab
            if hard:
                assert close(np.log(np.maximum(trace.comm_prob[sl, j], 1e-38)).astype(np.float64),
                             ep["logp"][..., comm_col]), lab
            at += L
        _assert_padding(trace, slice(t0, None), j)
    return compared


def _assert_padding(trace, rows, j):
    for k, v in trace.arrays().items():
        if k != "env_id":
            assert not v[rows, j].any(), k


@pytest.mark.parametrize("sampled", [True, False], ids=["sampled", "greedy"])
@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("B", [5, 13])
@pytest.mark.parametrize("case", sorted(ORACLE_CASES))
def test_trace_equals_the_oracle_replay(case, B, impl, sampled):
    name, max_steps = ORACLE_CASES[case]
    E = 2
    meta, z = load_golden(name)
    args, env, net, tr, p = episode_trainer(meta, B, impl=impl, eval_nenvs=B, max_steps=max_steps)
    stat, trace, cmap = tr.evaluate_trace(E, greedy=not sampled, slots=B)
    e = tr._eval["env"]
    assert stat["num_episodes"] == E * B
    T = E * max_steps
    assert trace.valid.shape == (T, B) and np.array_equal(trace.env_id, int(e.cfg.env_id0) + np.arange(B))
    if sampled:
        n = _trace_vs_oracle(args, z, p, trace, int(e.cfg.seed), E, True, case)
        assert n >= B // 2, (case, n)
    else:
        with greedy():
            _trace_vs_oracle(args, z, p, trace, int(e.cfg.seed), E, False, case)
    assert int(trace.valid.sum()) == stat["num_steps"]
    assert tr._eval["trace"].guards_intact()


def _twins(name, B, **over):
    return update_trainer(name, B, False, eval_nenvs=B, **over), update_trainer(name, B, False, eval_nenvs=B, **over)


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("name", [PP, TJ])
def test_recording_changes_nothing(name, use_graph):
    plain, rec = _twins(name, 256, use_graph=use_graph)
    same_stat(plain.evaluate(2), rec.evaluate(2))
    k_eval = rec._graphs.get("evaluate")
    for greedy_ in (False, True):
        same_stat(plain.evaluate(2, greedy_), rec.evaluate_trace(2, greedy_, slots=7)[0])
    same_stat(plain.evaluate(2), rec.evaluate(2))
    if use_graph:                         # evaluate replays the graph it captured before the recordings
        assert rec._graphs["evaluate"][1] is k_eval[1]
    for ep in range(2):
        same_stat(plain.train_batch(ep), rec.train_batch(ep))
    assert torch.equal(plain.optimizer.flat_params, rec.optimizer.flat_params)
    assert torch.equal(plain.env.env.tick, rec.env.env.tick)
    # row 0 of the full (h, c) records is allocated uninitialised and never written: every rollout starts with every
    # slot fresh, so the first policy step ignores the state it is handed there
    first_unwritten = ("rec_h", "rec_c")
    for k, v in plain._buf.items():
        if isinstance(v, torch.Tensor):
            a, b = (v[1:], rec._buf[k][1:]) if k in first_unwritten else (v, rec._buf[k])
            assert torch.equal(a, b), k


def _aggregate(tr, trace):
    """The comm map as numpy computes it from a trace of every slot."""
    e = tr._eval["env"]
    is_tj = tr.is_tj
    width, npos = (e.cfg.w, e.cfg.h * e.cfg.w) if is_tj else (e.cfg.dim, e.cfg.dim * e.cfg.dim)
    S = int(tr.args.max_steps)
    nf = e.cfg.N
    v = trace.valid.astype(bool)
    loc = trace.loc[:, :, :nf].astype(np.int64)
    rowmask = v[:, :, None] & (trace.alive[:, :, :nf] != 0)
    cell = loc[..., 0] * width + loc[..., 1]
    tep = np.broadcast_to(trace.t_ep[:, :, None].astype(np.int64), cell.shape)
    out = dict(visits=np.bincount(cell[rowmask], minlength=npos), visits_t=np.bincount(tep[rowmask], minlength=S))
    opened = None
    if tr.hard:
        opened = rowmask & (trace.action[:, :, :nf, -1] != 0)
        out.update(open=np.bincount(cell[opened], minlength=npos), open_t=np.bincount(tep[opened], minlength=S))
    if not is_tj:
        prey = trace.loc[:, :, nf:nf + 1].astype(np.int64)
        on = (loc == prey).all(-1).astype(np.int64)
        out["visits_reached"] = np.bincount(on[rowmask], minlength=2)
        if opened is not None:
            out["open_reached"] = np.bincount(on[opened], minlength=2)
    return out


MAP_CASES = {"pp_full": (PP, 8192, {}), "tj_full": (TJ, 4096, {}), "pp_1": (PP, 1024, dict(nagents=1, nfriendly=1)),
             "tj_1": (TJ, 1024, dict(nagents=1)), "pp_32": (PP, 1024, dict(nagents=31, nfriendly=31)),
             "tj_32": (TJ, 1024, dict(nagents=32))}


@pytest.mark.parametrize("case", sorted(MAP_CASES))
def test_comm_map_equals_the_trace(case):
    name, B, over = MAP_CASES[case]
    runs = []
    for _ in range(2):
        tr2 = update_trainer(name, B, False, eval_nenvs=B, max_steps=40, record_for_grad=False, **over)
        stat, trace, cmap = tr2.evaluate_trace(1, slots=B)
        runs.append((stat, trace, cmap))
        ref = _aggregate(tr2, trace)
        assert sorted(ref) == sorted(cmap), case
        for k in ref:
            assert np.array_equal(cmap[k].astype(np.int64), ref[k]), (case, k)
        assert int(cmap["visits_t"].sum()) > 0
    same_stat(runs[0][0], runs[1][0])
    for k, v in runs[0][1].arrays().items():
        assert np.array_equal(v, getattr(runs[1][1], k)), k
    for k in runs[0][2]:
        assert np.array_equal(runs[0][2][k], runs[1][2][k]), k


def _same_trace(a, b):
    (sa, ta, ca), (sb, tb, cb) = a, b
    same_stat(sa, sb)
    assert sorted(ta.arrays()) == sorted(tb.arrays())
    for k, v in ta.arrays().items():
        assert np.array_equal(v, getattr(tb, k)), k
    assert (ca is None) == (cb is None)
    for k in ca or {}:
        assert np.array_equal(ca[k], cb[k]), k


@pytest.mark.parametrize("name", [PP, TJ])
def test_graph_equals_eager(name):
    eager = update_trainer(name, 512, False, eval_nenvs=512)
    graph = update_trainer(name, 512, False, eval_nenvs=512, use_graph=True)
    keys = []
    for slots, cmap, greedy_ in ((8, True, False), (8, True, True), ([3, 100, 7], True, False), (8, False, False),
                                 (8, True, False)):
        _same_trace(eager.evaluate_trace(2, greedy_, slots=slots, comm_map=cmap),
                    graph.evaluate_trace(2, greedy_, slots=slots, comm_map=cmap))
        keys.append(graph._graphs["evaluate_trace"][0])
    assert keys[2] != keys[1] and keys[3] != keys[2] and keys[4] != keys[3]
    same_stat(eager.evaluate(2), graph.evaluate(2))


def test_random_policy_traces():
    _, tr = random_trainer(random_args("c2", nenvs=64, eval_nenvs=64, max_steps=20))
    ref = random_trainer(random_args("c2", nenvs=64, eval_nenvs=64, max_steps=20))[1]
    stat, trace, cmap = tr.evaluate_trace(2, slots=[0, 5, 63])
    same_stat(stat, ref.evaluate(2))
    assert trace.comm_prob is None and sorted(cmap) == ["visits", "visits_reached", "visits_t"]
    assert int(trace.valid.sum(0).min()) >= 2 and trace.done.sum() == 2 * 3
    assert int(cmap["visits_t"][0]) == 2 * 64 * tr.args.nagents
    assert tr._eval["trace"].guards_intact()


def test_without_hard_attn_the_map_has_visits_only():
    tr = update_trainer(PP, 128, False, eval_nenvs=128, record_for_grad=False, grad_impl="auto", **UPDATE_IC)
    stat, trace, cmap = tr.evaluate_trace(1, slots=4)
    assert trace.comm_prob is None
    assert sorted(cmap) == ["visits", "visits_reached", "visits_t"]
    assert int(cmap["visits_t"].sum()) == stat["num_steps"] * tr.args.nagents


def test_bad_slot_lists_raise_and_padding_is_zero():
    tr = update_trainer(PP, 64, False, eval_nenvs=64, max_steps=30, dim=5, nagents=3, nfriendly=3)
    for bad in ([1, 1], [64], [-1], 0, 65, []):
        with pytest.raises(ValueError):
            tr.evaluate_trace(1, slots=bad)
    stat, trace, cmap = tr.evaluate_trace(2, slots=64)
    assert tr._eval["trace"].guards_intact()
    pad = ~trace.valid.astype(bool)
    assert pad.any()                      # mixed mode: episodes end early, so slots finish their quota before T
    for k, v in trace.arrays().items():
        if k != "env_id":
            assert not v[pad].any(), k
    assert np.array_equal(trace.valid.sum(0), tr._eval["buf"]["stat_steps"].cpu().numpy())


def test_out_of_range_slot_raises_the_device_flag():
    """A slot list that bypasses the Python check reaches the kernel, which flags it instead of writing."""
    from ic3net_b200 import _lib
    tr = update_trainer(PP, 32, False, eval_nenvs=32, max_steps=10)
    tr.evaluate_trace(1, slots=4)
    rec = tr._eval["trace"]
    rec.t["slots"][2] = 32
    vec, e, _ = tr.evaluate_trace_vector(1, slots=4)
    assert int(vec[3].item()) & _lib.ERR_TRACE_SLOT
    assert rec.guards_intact()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_equal_one_process():
    here = os.path.dirname(os.path.abspath(__file__))
    B = 64
    with tempfile.TemporaryDirectory() as d:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
               "127.0.0.1", "--master-port", "29743", os.path.join(here, "eval_trace_nccl_worker.py"), d, str(B)]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600)
        assert r.returncode == 0, r.stdout.decode()[-4000:]
        ranks = [dict(np.load(os.path.join(d, "rank%d.npz" % k))) for k in range(2)]
    sys.path.insert(0, here)
    import eval_trace_nccl_worker as w
    _, tr = w.build(2 * B, 0)
    stat, _, cmap = tr.evaluate_trace(2, slots=2 * B)
    _, trace, _ = w.build(2 * B, 0)[1].evaluate_trace(2, slots=2 * B)
    for k, res in enumerate(ranks):
        assert int(res["num_steps"]) == stat["num_steps"] and int(res["num_episodes"]) == stat["num_episodes"]
        for key in cmap:
            assert np.array_equal(res["map_" + key], cmap[key]), key
        sl = slice(k * B, (k + 1) * B)
        assert np.array_equal(res["env_id"], trace.env_id[sl])
        for key, v in trace.arrays().items():
            if key != "env_id":
                assert np.array_equal(res[key], v[:, sl]), key


def test_cli_writes_one_trace_per_evaluation(tmp_path):
    from ic3net_b200 import main as cli
    base = ["--env_name", "predator_prey", "--nagents", "3", "--dim", "5", "--vision", "0", "--max_steps", "20",
            "--hid_size", "128", "--ic3net", "--recurrent", "--nenvs", "32", "--num_epochs", "2", "--epoch_size", "1",
            "--batch_size", "20", "--seed", "4", "--eval_every", "1", "--eval_nenvs", "16"]
    prefix = str(tmp_path / "tr")
    assert cli.main(base + ["--save", str(tmp_path / "a.pt"), "--eval_trace", prefix, "--eval_trace_slots", "5"]) == 0
    files = sorted(os.listdir(tmp_path))
    assert "tr_epoch1.npz" in files and "tr_epoch2.npz" in files
    z = np.load(prefix + "_epoch1.npz")
    T, K = 20, 5
    assert z["loc"].shape == (T, K, 4, 2) and z["loc_next"].shape == (T, K, 4, 2)
    assert z["action"].shape == (T, K, 3, 2) and z["comm_prob"].shape == (T, K, 3)
    for k in ("value", "reward", "alive"):
        assert z[k].shape == (T, K, 3), k
    for k in ("t_ep", "done", "success", "valid"):
        assert z[k].shape == (T, K), k
    assert z["env_id"].shape == (K,) and z["map_visits"].shape == (25,) and z["map_open_t"].shape == (20,)
    assert str(z["env_name"]) == "predator_prey" and list(z["grid_shape"]) == [5, 5] and int(z["max_steps"]) == 20
    assert cli.main(base + ["--save", str(tmp_path / "b.pt")]) == 0
    with cli._utils_alias():
        a = torch.load(str(tmp_path / "a.pt"), weights_only=False)
        b = torch.load(str(tmp_path / "b.pt"), weights_only=False)
    assert sorted(a) == sorted(b)
