"""GPU tests of the message recorder: Trainer.evaluate_trace(messages=True) (csrc/eval_trace.cu, ic3_trace_comm_step and
ic3_message_map_step) against the float64 oracle slot by slot, against its own trace, its message map against a numpy
aggregation of a trace of every slot, and recording messages changing nothing else.

Run as a script (under torch.distributed.run) this module is the two-rank worker of test_two_ranks_sum_their_maps."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from gpu_harness import (PP, ROW_TOL, TJ, UPDATE_IC, close, episode_trainer, ff_trainer, random_args, random_trainer,
                         same_stat, update_trainer)
from helpers import load_golden, make_oracle_env, tj_tables
from greedy_oracle import greedy
from oracle.rollout import run_episode

pytestmark = pytest.mark.gpu

# fixture, max_steps, argument overrides
ORACLE_CASES = {"pp_mixed": ("ep_pp_hard_ic3net", 30, {}), "pp_enemy": ("ep_pp_enemy_ic3net", 20, {}),
                "tj_hard": ("ep_tj_hard_ic3net", 30, {}),
                "pp_commnet_sum": ("ep_pp_hard_commnet", 30, dict(comm_mode="sum"))}
SCALE = 2.0 ** 32


def _messages_f64(h_in, g, alive, fresh, avg):
    """(m, S) of one lock-step of one slot in float64: m_j = h_j unless fresh or not alive; S_k = g_k sum_{j != k}
    g_j m_j, / (n_alive - 1) with avg and n_alive > 1 (every row is alive when fresh)."""
    n = len(g)
    live = np.zeros(n, bool) if fresh else alive.astype(bool)
    m = np.where(live[:, None], h_in, 0.0)
    n_alive = n if fresh else int(alive.astype(bool).sum())
    den = float(n_alive - 1) if avg and n_alive > 1 else 1.0
    gm = g.astype(np.float64)[:, None] * m
    S = g.astype(np.float64)[:, None] * (gm.sum(0)[None, :] - gm) / den
    return m, S


def _oracle_messages(args, z, p, trace, seed, E, label):
    """Replay every recorded slot on the oracle (its env following the recorded actions) and compare msg_h, msg_gate
    and msg_in with the float64 messages of the oracle's own hidden states."""
    is_tj = args.env_name == "traffic_junction"
    hard = bool(args.hard_attn) and bool(args.commnet)
    avg = getattr(args, "comm_mode", "avg") == "avg"
    n, H = args.nagents, args.hid_size
    # S sums up to n - 1 messages, each held to ROW_TOL against the oracle: with comm_mode sum their errors add up
    s_tol = ROW_TOL if avg else ROW_TOL * max(1, n - 1)
    for j, env_id in enumerate(trace.env_id):
        orc = make_oracle_env(args, tj_tables(z) if is_tj else None)
        t0 = 0
        for k in range(E):
            ep = run_episode(orc, p, args, seed, int(env_id), tick0=t0, episode=k,
                             forced_actions=trace.action[t0:t0 + args.max_steps, j].astype(np.int64))
            L = ep["num_steps"]
            lab = "%s slot %d episode %d" % (label, j, k)
            for t in range(L):
                h_in = np.zeros((n, H)) if t == 0 else ep["h"][t - 1]
                alive = ep["alive_in"][t]
                g = alive * (ep["comm_in"][t] if hard else 1)
                if t == 0:                               # fresh: alive = 1, comm_action = 0
                    g = np.zeros(n) if hard else np.ones(n)
                m, S = _messages_f64(h_in, g, alive, t == 0, avg)
                assert np.array_equal(trace.msg_gate[t0 + t, j], g.astype(np.uint8)), (lab, t)
                assert close(trace.msg_h[t0 + t, j], m), (lab, t)
                assert close(trace.msg_in[t0 + t, j], S, s_tol), (lab, t)
            assert not trace.msg_h[t0, j].any() and not trace.msg_in[t0, j].any(), lab
            t0 += L
        for key in ("msg_h", "msg_gate", "msg_in"):      # padding rows after the quota
            assert not getattr(trace, key)[t0:, j].any(), (label, j, key)


@pytest.mark.parametrize("sampled", [True, False], ids=["sampled", "greedy"])
@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("B", [5, 13])
@pytest.mark.parametrize("case", sorted(ORACLE_CASES))
def test_messages_equal_the_oracle_replay(case, B, impl, sampled):
    name, max_steps, over = ORACLE_CASES[case]
    E = 2
    meta, z = load_golden(name)
    args, env, net, tr, p = episode_trainer(meta, B, impl=impl, eval_nenvs=B, max_steps=max_steps, **over)
    stat, trace, cmap = tr.evaluate_trace(E, greedy=not sampled, slots=B, messages=True)
    e = tr._eval["env"]
    T = E * max_steps
    assert trace.msg_h.shape == (T, B, args.nagents, args.hid_size) and trace.msg_gate.shape == (T, B, args.nagents)
    if sampled:
        _oracle_messages(args, z, p, trace, int(e.cfg.seed), E, case)
    else:
        with greedy():
            _oracle_messages(args, z, p, trace, int(e.cfg.seed), E, case)
    if case == "tj_hard":                                # cars spawn and leave: dead rows are exercised
        assert (trace.valid[:, :, None].astype(bool) & (trace.alive == 0)).any()
    assert tr._eval["trace"].guards_intact()


def _fresh(trace):
    return trace.valid.astype(bool) & (trace.t_ep == 0)


def _check_own_trace(tr, trace, h_after):
    """msg_in from the recorded msg_h and msg_gate in float64, zero rows, and msg_h[t + 1] == h' of step t."""
    avg = getattr(tr.args, "comm_mode", "avg") == "avg"
    valid, fresh = trace.valid.astype(bool), _fresh(trace)
    T, K, NA, H = trace.msg_h.shape
    for t in range(T):
        for j in range(K):
            if not valid[t, j]:
                continue
            g = trace.msg_gate[t, j].astype(np.float64)
            n_alive = NA if fresh[t, j] else int((trace.alive[t, j] != 0).sum())
            den = float(n_alive - 1) if avg and n_alive > 1 else 1.0
            gm = g[:, None] * trace.msg_h[t, j].astype(np.float64)
            ref = g[:, None] * (gm.sum(0)[None, :] - gm) / den
            assert np.all(np.abs(trace.msg_in[t, j] - ref) <= 1e-6 * np.maximum(1.0, np.abs(ref))), (t, j)
    zero = fresh[:, :, None] | (trace.alive == 0) | ~valid[:, :, None]
    assert zero.any()
    assert not trace.msg_h[zero].any()
    assert not trace.msg_in[fresh].any() and not trace.msg_in[~valid].any() and not trace.msg_gate[~valid].any()
    # the hidden state a step leaves is what the next step sends, bit for bit
    carry = valid[1:, :, None] & ~fresh[1:, :, None] & (trace.alive[1:] != 0)
    assert carry.any()
    assert np.array_equal(trace.msg_h[1:][carry], h_after[:-1][carry])


OWN_CASES = {"pp": (PP, {}), "tj": (TJ, {}), "pp_enemy": (PP, dict(enemy_comm=True, nagents=11, nfriendly=10)),
             "pp_commnet_sum": (PP, dict(hard_attn=False, ic3net=False, comm_mode="sum"))}


@pytest.mark.parametrize("case", sorted(OWN_CASES))
def test_messages_agree_with_their_trace(case):
    name, over = OWN_CASES[case]
    tr = update_trainer(name, 48, False, eval_nenvs=48, max_steps=30, record_for_grad=False, **over)
    K = 12
    tr.evaluate_trace(2, slots=K, messages=True)
    rec = tr._eval["trace"]
    b = tr._eval["buf"]
    NA, H = tr.args.nagents, tr.args.hid_size
    slots = list(rec.slots)
    h_after = []
    step = rec.step

    def keep_h(t, s):                                    # between policy step t and env step t: h holds h'
        step(t, s)
        h_after.append(b["h"].view(-1, NA, H)[slots].cpu().numpy())
    rec.step = keep_h                                    # this recorder only (eager: run in stream order)
    stat, trace, cmap = tr.evaluate_trace(2, slots=K, messages=True)
    assert tr._eval["trace"] is rec and len(h_after) == trace.valid.shape[0]
    _check_own_trace(tr, trace, np.stack(h_after))
    assert rec.guards_intact()


def _keyed_sum(keys, vals, n):
    """out[k] = sum of vals[i] with keys[i] == k, int64 (exact in any order)."""
    out = np.zeros((n,) + vals.shape[1:], np.int64)
    if len(keys):
        order = np.argsort(keys, kind="stable")
        ks, vs = keys[order], vals[order]
        starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
        out[ks[starts]] = np.add.reduceat(vs, starts, axis=0)
    return out


def _aggregate_messages(tr, trace):
    """The message map as numpy computes it from a trace of every slot, with the rint(v * 2^32) int64 rule."""
    e = tr._eval["env"]
    is_tj = tr.is_tj
    width, P = (e.cfg.w, e.cfg.h * e.cfg.w) if is_tj else (e.cfg.dim, e.cfg.dim * e.cfg.dim)
    S = int(tr.args.max_steps)
    R = P + S + (0 if is_tj else 2)
    nf = e.cfg.N
    H = trace.msg_h.shape[-1]
    sent, recv, senders = np.zeros((R, H), np.int64), np.zeros((R, H), np.int64), np.zeros(R, np.int64)
    for t in range(trace.valid.shape[0]):                # one lock-step at a time keeps the host memory small
        rows = trace.valid[t].astype(bool)[:, None] & (trace.alive[t, :, :nf] != 0)
        loc = trace.loc[t, :, :nf].astype(np.int64)
        keys = [loc[..., 0] * width + loc[..., 1], np.broadcast_to(P + trace.t_ep[t].astype(np.int64)[:, None],
                                                                   rows.shape)]
        if not is_tj:
            keys.append(P + S + (loc == trace.loc[t, :, nf:nf + 1].astype(np.int64)).all(-1).astype(np.int64))
        open_ = rows & (trace.msg_gate[t, :, :nf] != 0)
        h = np.rint(trace.msg_h[t, :, :nf][open_].astype(np.float64) * SCALE).astype(np.int64)
        s = np.rint(trace.msg_in[t, :, :nf][rows].astype(np.float64) * SCALE).astype(np.int64)
        for key in keys:
            sent += _keyed_sum(key[open_], h, R)
            recv += _keyed_sum(key[rows], s, R)
            senders += np.bincount(key[open_], minlength=R)
    out = {}
    parts = [("", slice(0, P)), ("_t", slice(P, P + S))] + ([] if is_tj else [("_reached", slice(P + S, R))])
    for suffix, sl in parts:
        out["msg_sent" + suffix], out["msg_recv" + suffix], out["msg_senders" + suffix] = sent[sl], recv[sl], senders[sl]
    return out


MAP_CASES = {"pp_full": (PP, 8192, {}), "tj_full": (TJ, 4096, {}), "pp_1": (PP, 1024, dict(nagents=1, nfriendly=1)),
             "tj_1": (TJ, 1024, dict(nagents=1)), "pp_32": (PP, 1024, dict(nagents=31, nfriendly=31)),
             "tj_32": (TJ, 1024, dict(nagents=32))}


@pytest.mark.parametrize("case", sorted(MAP_CASES))
def test_message_map_equals_the_trace(case):
    """Eager and graph: each map equals the numpy aggregation of its own trace of every slot, and the two are equal."""
    name, B, over = MAP_CASES[case]
    runs = []
    for use_graph in (False, True):
        tr = update_trainer(name, B, False, eval_nenvs=B, max_steps=20, record_for_grad=False, use_graph=use_graph,
                            **over)
        stat, trace, cmap = tr.evaluate_trace(1, slots=B, messages=True)
        ref = _aggregate_messages(tr, trace)
        for k in ref:
            assert np.array_equal(cmap[k], ref[k]), (case, k)
        assert int(cmap["msg_senders_t"].sum()) > 0 and np.abs(cmap["msg_sent_t"]).sum() > 0
        if tr.args.nagents > 1:                          # a lone agent receives nothing
            assert np.abs(cmap["msg_recv_t"]).sum() > 0
        assert tr._eval["trace"].guards_intact()
        runs.append((stat, cmap))
        del trace, tr
    same_stat(runs[0][0], runs[1][0])
    for k, v in runs[0][1].items():
        assert np.array_equal(v, runs[1][1][k], equal_nan=True), k


def _same(a, b):
    (sa, ta, ca), (sb, tb, cb) = a, b
    same_stat(sa, sb)
    assert sorted(ta.arrays()) == sorted(tb.arrays())
    for k, v in ta.arrays().items():
        assert np.array_equal(v, getattr(tb, k)), k
    assert sorted(ca or {}) == sorted(cb or {})
    for k in ca or {}:
        assert np.array_equal(ca[k], cb[k], equal_nan=True), k


@pytest.mark.parametrize("name", [PP, TJ])
def test_graph_equals_eager(name):
    eager = update_trainer(name, 512, False, eval_nenvs=512)
    graph = update_trainer(name, 512, False, eval_nenvs=512, use_graph=True)
    keys = []
    for slots, cmap, msg in ((8, True, True), ([3, 100, 7], True, True), (8, False, True), (8, True, False),
                             (8, True, True)):
        _same(eager.evaluate_trace(2, slots=slots, comm_map=cmap, messages=msg),
              graph.evaluate_trace(2, slots=slots, comm_map=cmap, messages=msg))
        keys.append(graph._graphs["evaluate_trace"][0])
    assert keys[3] != keys[4] and keys[2] != keys[3]
    same_stat(eager.evaluate(2), graph.evaluate(2))


def _twins(name, B, **over):
    return update_trainer(name, B, False, eval_nenvs=B, **over), update_trainer(name, B, False, eval_nenvs=B, **over)


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("name", [PP, TJ])
def test_messages_change_nothing(name, use_graph):
    plain, rec = _twins(name, 256, use_graph=use_graph)
    same_stat(plain.evaluate(2), rec.evaluate_trace(2, slots=7, messages=True)[0])
    a = plain.evaluate_trace(2, slots=7)
    b = rec.evaluate_trace(2, slots=7, messages=True)
    same_stat(a[0], b[0])
    assert b[1].msg_h is not None and a[1].msg_h is None
    for k, v in a[1].arrays().items():
        assert np.array_equal(v, getattr(b[1], k)), k
    for k in a[2]:
        assert np.array_equal(a[2][k], b[2][k]), k
    assert not (set(b[2]) - set(a[2])) - {k for k in b[2] if k.startswith("msg_")}
    assert rec._eval["trace"].guards_intact()
    for ep in range(2):
        same_stat(plain.train_batch(ep), rec.train_batch(ep))
    assert torch.equal(plain.optimizer.flat_params, rec.optimizer.flat_params)
    assert torch.equal(plain.env.env.tick, rec.env.env.tick)


def test_refusals():
    cases = [("comm_passes 2", lambda: update_trainer(PP, 16, False, eval_nenvs=16, init_seed="fixture", comm_passes=2,
                                                      share_weights=False)),
             ("models.MLP", lambda: ff_trainer(PP, 16, "mlp", eval_nenvs=16)),
             ("non-recurrent CommNet", lambda: ff_trainer(PP, 16, "ic3net", eval_nenvs=16)),
             ("models.RNN", lambda: update_trainer(PP, 16, False, eval_nenvs=16, record_for_grad=False, **UPDATE_IC)),
             ("comm_mask_zero", lambda: update_trainer(PP, 16, False, eval_nenvs=16, comm_mask_zero=True)),
             ("models.Random", lambda: random_trainer(random_args("c2", nenvs=16, eval_nenvs=16, max_steps=20))[1])]
    for label, make in cases:
        tr = make()
        with pytest.raises(NotImplementedError):
            tr.evaluate_trace(1, slots=2, messages=True)
        ev = getattr(tr, "_eval", None)                  # refused before any device work
        assert ev is None or ev.get("trace") is None, label
        tr.evaluate_trace(1, slots=2)                    # the recording without messages still runs


def test_bad_slots_raise():
    tr = update_trainer(PP, 32, False, eval_nenvs=32, max_steps=10)
    for bad in ([1, 1], [32], [-1], 0, 33, []):
        with pytest.raises(ValueError):
            tr.evaluate_trace(1, slots=bad, messages=True)
    from ic3net_b200 import _lib
    tr.evaluate_trace(1, slots=4, messages=True)
    rec = tr._eval["trace"]
    rec.t["slots"][2] = 32                               # past the Python check: the kernels flag it
    vec, e, _ = tr.evaluate_trace_vector(1, slots=4, messages=True)
    assert int(vec[3].item()) & _lib.ERR_TRACE_SLOT
    assert rec.guards_intact()


# ---------------------------------------------------------------------------------------------------- two ranks

def _worker_trainer(B, rank):
    from ic3net_b200.multi_gpu import MultiGPUTrainer
    tr = update_trainer(PP, B, False, eval_nenvs=B, env_id0=rank * B, max_steps=20, record_for_grad=False)
    return MultiGPUTrainer(tr.args, lambda: tr)


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_sum_their_maps():
    B = 64
    with tempfile.TemporaryDirectory() as d:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
               "127.0.0.1", "--master-port", "29751", os.path.abspath(__file__), d, str(B)]
        here = os.path.dirname(os.path.abspath(__file__))
        env = dict(os.environ, PYTHONPATH=os.pathsep.join([here, os.path.dirname(here),
                                                           os.environ.get("PYTHONPATH", "")]))
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, env=env)
        assert r.returncode == 0, r.stdout.decode()[-4000:]
        ranks = [dict(np.load(os.path.join(d, "rank%d.npz" % k))) for k in range(2)]
    for key in ranks[0]:
        if key.startswith("sum_"):
            own = ranks[0]["own_" + key[4:]] + ranks[1]["own_" + key[4:]]
            assert np.array_equal(ranks[0][key], own) and np.array_equal(ranks[1][key], own), key


def _worker_main(out, B):
    import torch.distributed as dist
    rank = int(os.environ["RANK"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
    mt = _worker_trainer(B, rank)
    _, _, own = mt.trainer.evaluate_trace(1, slots=4, messages=True)
    mt.trainer._eval = None                              # the same episodes again, now summed over ranks
    _, _, summed = mt.evaluate_trace(1, slots=4, messages=True)
    keys = [k for k in own if k.startswith("msg_") and own[k].dtype == np.int64]
    np.savez(os.path.join(out, "rank%d.npz" % rank), **{"own_" + k: own[k] for k in keys},
             **{"sum_" + k: summed[k] for k in keys})
    dist.destroy_process_group()


if __name__ == "__main__":
    _worker_main(sys.argv[1], int(sys.argv[2]))


# ---------------------------------------------------------------------------------------------------- command line

def test_cli_writes_the_messages(tmp_path):
    from ic3net_b200 import main as cli
    base = ["--env_name", "predator_prey", "--nagents", "3", "--dim", "5", "--vision", "0", "--max_steps", "20",
            "--hid_size", "128", "--ic3net", "--recurrent", "--nenvs", "32", "--num_epochs", "1", "--epoch_size", "1",
            "--batch_size", "20", "--seed", "4", "--eval_every", "1", "--eval_nenvs", "16", "--eval_trace_slots", "5"]
    with_msg, without = str(tmp_path / "m"), str(tmp_path / "p")
    assert cli.main(base + ["--eval_trace", with_msg, "--eval_trace_messages"]) == 0
    assert cli.main(base + ["--eval_trace", without]) == 0
    zm, zp = dict(np.load(with_msg + "_epoch1.npz")), dict(np.load(without + "_epoch1.npz"))
    T, K, H = 20, 5, 128
    assert zm["msg_h"].shape == (T, K, 3, H) and zm["msg_in"].shape == (T, K, 3, H) and zm["msg_gate"].shape == (T, K, 3)
    assert zm["map_msg_sent"].shape == (25, H) and zm["map_msg_recv_t"].shape == (20, H)
    assert zm["map_msg_senders_reached"].shape == (2,) and float(zm["map_msg_scale"]) == 2.0 ** -32
    assert int(zm["hid_size"]) == H
    new = {k for k in zm if k.startswith("msg_") or k.startswith("map_msg_")} | {"hid_size"}
    assert sorted(zp) == sorted(set(zm) - new)
    today = {"loc", "loc_next", "alive", "action", "value", "reward", "t_ep", "done", "success", "valid", "comm_prob",
             "env_id", "map_visits", "map_open", "map_visits_t", "map_open_t", "map_visits_reached",
             "map_open_reached", "env_name", "grid_shape", "nagents", "nfriendly", "naction_heads", "max_steps",
             "episodes", "greedy", "hard_attn"}
    assert set(zp) == today
    with pytest.raises(SystemExit):
        cli.main(base + ["--eval_trace_messages"])
