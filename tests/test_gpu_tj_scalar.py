"""GPU tests of the traffic junction with ``vocab_type='scalar'`` (csrc/tj_env.cu, the index / dense encoders of
csrc/policy.cu and csrc/tj_env.cu, both policy kernels) against the fixtures the unmodified reference produced
(tests/golden/tj_scalar_*.npz, scripts/gen_golden_tj_scalar.py) and the float64 step of tests/policy_ref.py.

Bars: bit-exact states, masks and observations, rewards equal to float32(reference); every encoder form gives the same x
bit for bit; policy outputs within 1e-5 * max(1, |ref|) (DESIGN.md section 2); gradients within 2e-3 of the reference's
compute_grad, as for the bool vocabulary."""
import ctypes as C

import numpy as np
import pytest
import torch

from gpu_harness import LOSS_ATOL, LOSS_RTOL, close, cpu, episode_trainer, trainer_rows
from helpers import load_golden, ns, tj_tables
from tj_scalar_oracle import make_env as make_oracle

pytestmark = pytest.mark.gpu
ENV_CASES = ["tj_scalar_env_easy", "tj_scalar_env_medium_v1", "tj_scalar_env_hard"]
EP = "tj_scalar_ep_medium_ic3net"
GRAD = "tj_scalar_grad_hard_ic3net_h128"


def lib():
    from ic3net_b200 import _lib
    return _lib, _lib.load()


def other_writers(env):
    """The observation of the env's current state from ic3_tj_obs and from the persistent writer ic3_tj_obs_bounded."""
    _lib, L = lib()
    a, b = env._new_obs(), env._new_obs()
    _lib.check(L.ic3_tj_obs(C.byref(env.cfg), C.byref(env.state), a.data_ptr(), _lib.stream()))
    _lib.check(L.ic3_tj_obs_bounded(C.byref(env.cfg), C.byref(env.state), b.data_ptr(), _lib.stream()))
    return a, b


@pytest.mark.parametrize("name", ENV_CASES)
def test_env_matches_reference_fixture(name):
    """One env on the fixture's Philox streams: states and rewards of the step kernel, and the observation from the step
    kernel, ic3_tj_obs, the side-stream writer and a LazyObs handle, all bit for bit the reference's."""
    from ic3net_b200 import data
    meta, z = load_golden(name)
    args = ns(meta["args"], nenvs=1, seed=meta["seed"], env_id0=meta["env_id"])
    w = data.init(args.env_name, args)
    env = w.env
    assert w.observation_dim == meta["obs_dim"] == 4 + (2 * args.vision + 1) ** 2 * 2
    assert env.obs_layout == (0, 0, 0) and not hasattr(env, "BASE")
    obs = w.reset(0)
    assert np.array_equal(cpu(obs)[0], z["obs0"].astype(np.float32))
    for t in range(len(z["act"])):
        obs, r, done, info = w.step([z["act"][t][None]])
        aux = np.stack([cpu(env.wait)[0], cpu(env.route_id)[0], cpu(env.car_last_act)[0], cpu(env.car_route_loc)[0]], 1)
        assert np.array_equal(cpu(env.car_loc)[0], z["loc"][t]), (name, t)
        assert np.array_equal(aux, z["aux"][t]), (name, t)
        assert np.array_equal(cpu(info["alive_mask"])[0], z["alive"][t])
        assert np.array_equal(cpu(info["is_completed"])[0], z["completed"][t])
        assert np.array_equal(cpu(r)[0], z["reward"][t].astype(np.float32)), (name, t)
        assert np.array_equal(cpu(obs)[0], z["obs"][t]), (name, t)
        a, b = other_writers(env)
        torch.cuda.synchronize()
        assert torch.equal(a, obs) and torch.equal(b, obs), (name, t)
        env.obs_api = "handle"
        assert torch.equal(env._obs_handle().dense(), obs)
        env.obs_api = "dense"
    assert w.get_stat().get("success", -1) == meta["success"]


def test_batched_envs_match_oracle():
    """37 envs with distinct Philox streams against 37 oracle instances, random actions, vision 1."""
    from ic3net_b200 import data
    meta, z = load_golden("tj_scalar_env_medium_v1")
    B, seed, id0 = 37, 99, 5
    args = ns(meta["args"], nenvs=B, seed=seed, env_id0=id0)
    w = data.init(args.env_name, args)
    env = w.env
    orcs = [make_oracle(args, tj_tables(z)) for _ in range(B)]
    obs = cpu(w.reset(0))
    for b in range(B):
        assert np.array_equal(obs[b], orcs[b].reset(0).astype(np.float32))
    rs = np.random.RandomState(3)
    for t in range(40):
        act = rs.randint(0, 2, size=(B, args.nagents))
        obs, r, _, _ = w.step([torch.as_tensor(act)])
        obs, r = cpu(obs), cpu(r)
        for b in range(B):
            oo, orr, _, _ = orcs[b].step(act[b], seed=seed, env_id=id0 + b)
            assert np.array_equal(obs[b], oo.astype(np.float32)), (t, b)
            assert np.array_equal(r[b], orr.astype(np.float32)), (t, b)
            assert np.array_equal(cpu(env.car_loc)[b], orcs[b].car_loc)


@pytest.mark.parametrize("H", [32, 128])
def test_index_and_fused_encoders_equal_the_dense_encoder(H):
    """x from ic3_tj_encoder_index (env state) and from ic3_tj_obs_encode (observation written and encoded in one
    kernel) equals ic3_encoder_dense on the observation tensor bit for bit, with live and dead cars on the board."""
    import argparse
    from ic3net_b200 import data
    from ic3net_b200.comm import CommNetMLP
    _lib, L = lib()
    meta, _ = load_golden("tj_scalar_env_medium_v1")
    B = 300
    args = ns(meta["args"], nenvs=B, seed=7, env_id0=0)
    w = data.init(args.env_name, args)
    env = w.env
    w.reset(0)
    rs = np.random.RandomState(1)
    for _ in range(12):
        w.step([torch.as_tensor(rs.randint(0, 2, size=(B, args.nagents)))])
    alive = cpu(env.alive_mask)
    assert 0 < alive.mean() < 1
    pa = argparse.Namespace(nagents=args.nagents, hid_size=H, comm_passes=1, recurrent=True, rnn_type="LSTM",
                            continuous=False, naction_heads=[2, 2], comm_mask_zero=False, comm_mode="avg",
                            hard_attn=True, comm_init="uniform", share_weights=False, seed=0, env_id0=0, commnet=True,
                            policy_impl="simt")
    torch.manual_seed(0)
    net = CommNetMLP(pa, w.observation_dim)
    net.set_obs_layout(*env.obs_layout)
    cfg, wp = net.policy_cfg(B), net.packed()
    R = B * args.nagents
    obs, obs2 = env._get_obs(), env._new_obs()
    x_dense, x_index, x_fused = (torch.empty(R, H, device="cuda") for _ in range(3))
    _lib.check(L.ic3_encoder_dense(C.byref(cfg), C.byref(wp), obs.data_ptr(), x_dense.data_ptr(), _lib.stream()))
    _lib.check(L.ic3_tj_encoder_index(C.byref(env.cfg), C.byref(env.state), C.byref(cfg), C.byref(wp),
                                      x_index.data_ptr(), _lib.stream()))
    _lib.check(L.ic3_tj_obs_encode(C.byref(env.cfg), C.byref(env.state), C.byref(cfg), C.byref(wp), obs2.data_ptr(),
                                   x_fused.data_ptr(), _lib.stream()))
    torch.cuda.synchronize()
    assert torch.equal(obs2, obs)
    assert torch.equal(x_index, x_dense) and torch.equal(x_fused, x_dense)
    want = obs.reshape(R, -1).double() @ net.encoder.weight.detach().double().t() + net.encoder.bias.detach().double()
    assert float((x_dense.double() - want).abs().max()) < 1e-5
    dead = torch.as_tensor(alive.reshape(-1) == 0, device="cuda")
    assert torch.equal(x_dense[dead], net.encoder.bias.detach().expand(int(dead.sum()), H))


@pytest.mark.parametrize("obs_mode", ["index", "dense"])
@pytest.mark.parametrize("impl", ["tc", "simt"])
def test_episode_matches_reference_fixture(obs_mode, impl):
    """The reference's IC3Net episodes (vision 1) through the lock-step rollout on both policy kernels: actions, rewards,
    masks, values and log-probabilities."""
    meta, z = load_golden(EP)
    ids = meta["env_ids"]
    args, env, net, tr, _ = episode_trainer(meta, max(ids) + 1, obs_mode, impl=impl)
    assert not net.fuses_encoder(env.env) and net.encoder_table(env.env) is None
    assert not tr._overlap_obs()
    batch = tr.rollout(args.max_steps, meta["epoch"])
    torch.cuda.synchronize()
    checked = 0
    for i, env_id in enumerate(ids):
        g = lambda k: z["e%d_%s" % (i, k)]
        n = len(g("act"))
        act = cpu(batch.action)[:n, env_id]
        assert not ((act != g("act")) & (g("margin") > 1e-4)).any(), env_id
        if not np.array_equal(act, g("act")):
            continue                # an fp32-borderline draw flipped: the full-size test below covers the slot
        assert np.array_equal(cpu(batch.reward)[:n, env_id], g("reward").astype(np.float32))
        assert np.array_equal(cpu(batch.alive_mask)[:n, env_id], g("alive"))
        assert np.array_equal(cpu(batch.episode_mini_mask)[:n, env_id], g("mini"))
        assert close(cpu(batch.value)[:n, env_id], g("value"))
        lp = np.concatenate([g("logp%d" % k) for k in range(len(meta["heads"]))], -1)
        assert close(cpu(batch.logp)[:n, env_id], lp)
        checked += 1
    assert checked >= 1


@pytest.mark.parametrize("impl", ["tc", "simt"])
def test_full_size_every_row_matches_float64(impl):
    """Traffic-junction hard, 4096 slots x 20 cars: a 14-step rollout with max_steps 6 (every slot resets twice, cars
    spawn, crash, leave and sit dead at (0,0)); every row of every step against the float64 step on the observation
    rebuilt from the recorded env state (Trainer._record_state: loc, alive, last_act, route_id)."""
    meta, _ = load_golden(GRAD)
    args, env, net, tr, _ = episode_trainer(meta, 4096, impl=impl, seed=5, record_for_grad=True, grad_window=1, max_steps=6)
    assert not tr.grad_kernels
    trainer_rows(tr, 14, "tj scalar hard %s" % impl)
    alive = cpu(tr._buf["s_alive"])
    assert 0 < alive.mean() < 1


@pytest.mark.parametrize("impl", ["tc", "simt"])
def test_autograd_gradient_matches_the_reference(impl):
    """One slot on the fixture's streams stops at the reference's batch boundary and the autograd recompute (observations
    rebuilt from the records by ic3_tj_obs) gives the reference's compute_grad gradient."""
    meta, z = load_golden(GRAD)
    args, env, net, tr, _ = episode_trainer(meta, 1, impl=impl, env_id0=meta["env_id"], record_for_grad=True,
                                            grad_window=16, grad_impl="auto")
    assert tr.grad_impl == "autograd" and not tr.grad_kernels
    batch, stat = tr.run_batch(0)
    if stat["num_steps"] != meta["num_steps"]:
        pytest.skip("an fp32-borderline draw flipped an action of this trajectory (the full-size test covers it)")
    assert stat["num_episodes"] == meta["num_episodes"]
    tr.optimizer.zero_grad(set_to_none=False)
    s = tr.compute_grad(batch)
    for q in ("action_loss", "value_loss", "entropy"):
        assert np.isclose(s[q], meta[q], rtol=LOSS_RTOL, atol=LOSS_ATOL), (q, s[q], meta[q])
    checked = 0
    for key, prm in net.named_parameters():
        if "g_" + key in z.files:
            want = z["g_" + key]
            assert np.abs(cpu(prm.grad) - want).max() <= 2e-3 * max(np.abs(want).max(), 1e-30), key
            checked += 1
        elif "gsample_" + key in z.files:
            got = cpu(prm.grad).astype(np.float64).ravel()
            ws = z["gsample_" + key]
            assert np.abs(got[::max(1, got.size // 2048)][:2048] - ws).max() <= 2e-3 * max(np.abs(ws).max(), 1e-30), key
            checked += 1
    assert checked >= 8


@pytest.mark.parametrize("grad_impl", ["kernels", "kernels_ff"])
def test_gradient_kernels_refuse_the_scalar_vocabulary(grad_impl):
    meta, _ = load_golden(GRAD)
    # kernels_ff: the non-recurrent CommNet it would cover on the bool vocabulary
    kw = dict(recurrent=False, rnn_type="MLP", commnet=True, ic3net=False, hard_attn=False, comm_action_one=False) \
        if grad_impl == "kernels_ff" else {}
    m = dict(meta, args=dict(meta["args"], **kw))
    with pytest.raises(NotImplementedError):
        episode_trainer(m, 4, impl="tc" if grad_impl == "kernels" else "simt", weights=False, record_for_grad=True,
                        grad_window=16, grad_impl=grad_impl)


@pytest.mark.parametrize("obs_mode", ["index", "dense"])
def test_graph_replay_equals_eager(obs_mode):
    meta, _ = load_golden(EP)
    res = {}
    for use_graph in (True, False):
        args, env, net, tr, _ = episode_trainer(meta, 16, obs_mode, impl="tc", seed=5, use_graph=use_graph)
        out = []
        for _ in range(3):
            b = tr.rollout(40, 0)
            torch.cuda.synchronize()
            out.append((cpu(b.action).copy(), cpu(b.reward).copy(), cpu(b.value).copy()))
        res[use_graph] = out
    for a, b in zip(res[True], res[False]):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))


def test_cli_trains_the_scalar_vocabulary(capsys):
    from ic3net_b200 import main as cli
    rc = cli.main(["--env_name", "traffic_junction", "--vocab_type", "scalar", "--nagents", "5", "--dim", "6",
                   "--vision", "1", "--max_steps", "20", "--difficulty", "easy", "--add_rate_min", "0.3",
                   "--add_rate_max", "0.3", "--hid_size", "128", "--ic3net", "--recurrent", "--nenvs", "64",
                   "--num_epochs", "2", "--epoch_size", "1", "--batch_size", "40"])
    out = capsys.readouterr().out
    assert rc == 0 and "Epoch" in out, out[-2000:]
