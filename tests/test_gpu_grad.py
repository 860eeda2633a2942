"""GPU parity tests of the gradient row (SURVEY 8(f)-1): the returns-scan kernel and
``Trainer.compute_grad`` against the float64 oracle (oracle/grad.py), which is itself pinned to the
reference's ``Trainer.compute_grad`` (tests/golden/grad_*.npz).  Every env slot plays one reference
process; the expected gradient is the SUM over slots (multi_processing.py:92-94)."""
import numpy as np
import pytest
import torch

from bptt_ref import oracle_grad_sum
from helpers import finish_args, golden_names, load_golden, ns
from oracle import grad as ograd
from oracle import policy as opolicy
from oracle.gen_golden import make_weights

pytestmark = pytest.mark.gpu


def cpu(t):
    return t.detach().cpu().numpy()


def test_returns_scan_matches_oracle():
    import ctypes as C
    from ic3net_b200 import _lib
    rs = np.random.RandomState(0)
    T, B, N = 37, 9, 5
    reward = rs.randn(T, B, N).astype(np.float32)
    emask = (rs.rand(T, B) > 0.15).astype(np.uint8)
    mini = (rs.rand(T, B, N) > 0.2).astype(np.uint8)
    for gamma, mr in ((1.0, 0.0), (0.9, 1.0), (0.97, 0.4)):
        out = torch.empty(T, B, N, device="cuda")
        r, e, m = (torch.tensor(x, device="cuda") for x in (reward, emask, mini))
        _lib.check(_lib.load().ic3_returns_scan(T, B, N, gamma, mr, r.data_ptr(), e.data_ptr(), m.data_ptr(),
                                                out.data_ptr(), _lib.stream()))
        for b in range(B):
            want = ograd.returns_np(reward[:, b].astype(np.float64), np.repeat(emask[:, b, None], N, 1).astype(float),
                                    mini[:, b].astype(float), np.float32(gamma).item(), np.float32(mr).item())
            assert np.allclose(cpu(out)[:, b], want, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("name", golden_names("grad_"))
@pytest.mark.parametrize("impl,grad_impl", [("tc", "kernels"), ("tc", "autograd"), ("tc", "manual"), ("simt", "autograd")])
def test_compute_grad_matches_oracle(name, impl, grad_impl):
    from ic3net_b200 import data
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    meta, z = load_golden(name)
    B, seed, id0 = 5, 808, 30
    args = ns(meta["args"], nenvs=B, seed=seed, env_id0=id0, obs_mode="index", use_graph=False, policy_impl=impl,
              record_for_grad=True, grad_window=16, grad_impl=grad_impl)
    if impl == "tc" and args.hid_size != 128:
        pytest.skip("tensor-core path (and the BPTT kernels) are specialised for hid_size 128")
    env = data.init(args.env_name, args)
    finish_args(args, env)
    net = CommNetMLP(args, args.num_inputs)
    sd = make_weights(meta["weights_seed"], args.num_inputs, args.hid_size, args.naction_heads, args.comm_init)
    net.load_state_dict({k: torch.from_numpy(v).float() for k, v in sd.items()})
    tr = Trainer(args, net, env)
    batch, stat = tr.run_batch(0)
    T, quota = tr.batch_plan()
    assert quota == args.batch_size
    tr.optimizer.zero_grad(set_to_none=False)
    s = tr.compute_grad(batch)
    # ---- oracle: every slot is one reference process ----
    p = opolicy.params_to_f64(sd)
    want, wstat, nsteps_total = oracle_grad_sum(args, z, p, cpu(batch.action), cpu(batch.valid), seed, id0, quota, T)
    for q in wstat:
        assert np.isclose(s[q], wstat[q], rtol=2e-4, atol=1e-3), (q, s[q], wstat[q])
    assert stat["num_steps"] == nsteps_total
    worst = 0.0
    for key, prm in net.named_parameters():
        if want[key] is None or not np.any(want[key]):
            assert prm.grad is None or float(prm.grad.abs().max()) == 0.0, key
            continue
        err = np.abs(cpu(prm.grad) - want[key]).max() / np.abs(want[key]).max()
        worst = max(worst, err)
        assert err < 2e-3, (name, key, err)
    assert tr.grad_kernels == (grad_impl == "kernels")
    print(name, impl, grad_impl, "worst relative gradient error %.2e" % worst)
    assert worst < (1e-4 if grad_impl == "kernels" else 2e-3)


def test_train_batch_updates_parameters():
    from ic3net_b200 import data
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    meta, z = load_golden("grad_pp_easy_ic3net")
    args = ns(meta["args"], nenvs=64, seed=3, env_id0=0, obs_mode="index", use_graph=False, record_for_grad=True)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    net = CommNetMLP(args, args.num_inputs)
    tr = Trainer(args, net, env)
    before = [p.detach().clone() for p in tr.params]
    stat = tr.train_batch(0)
    assert 64 * args.batch_size <= stat["num_steps"] <= 64 * tr.steps_per_batch()
    assert all(np.isfinite(stat[k]) for k in ("action_loss", "value_loss", "entropy"))
    changed = [not torch.equal(a, b) for a, b in zip(before, tr.params)]
    names = [n for n, _ in net.named_parameters()]
    for n, c in zip(names, changed):
        assert c == (not n.startswith("hidd_encoder")), n      # the unused module gets no gradient (comm.py:57)
    stat2 = tr.train_batch(1)                                  # re-packed weights, second update runs
    assert 64 * args.batch_size <= stat2["num_steps"] <= 64 * tr.steps_per_batch()


@pytest.mark.parametrize("grad_impl", ["auto", "autograd"])
@pytest.mark.parametrize("name", golden_names("grad_"))
def test_run_batch_boundary_and_gradient_match_the_reference(name, grad_impl):
    """SURVEY a20 / f-1 against numbers the UNMODIFIED reference produced: the fixture is one reference worker
    (`Trainer.run_batch` + `compute_grad`, trainer.py:227-242,128-225) whose draws were routed to the Philox streams
    of (seed, env_id).  One GPU slot with the same streams must stop at the same batch boundary (whole episodes
    until >= batch_size steps: `num_steps`, `num_episodes`), see the same returns, and produce the same gradient."""
    from ic3net_b200 import data
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    meta, z = load_golden(name)
    args = ns(meta["args"], nenvs=1, seed=meta["seed"], env_id0=meta["env_id"], obs_mode="index", use_graph=False,
              record_for_grad=True, grad_window=16, grad_impl=grad_impl)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    net = CommNetMLP(args, args.num_inputs)
    sd = make_weights(meta["weights_seed"], args.num_inputs, args.hid_size, args.naction_heads, args.comm_init)
    net.load_state_dict({k: torch.from_numpy(v).float() for k, v in sd.items()})
    tr = Trainer(args, net, env)
    batch, stat = tr.run_batch(0)
    if stat["num_steps"] != meta["num_steps"]:
        # only an fp32-borderline action draw can send the free-running slot onto another trajectory
        pytest.skip("an fp32-borderline draw flipped an action of this trajectory (teacher-forced test covers it)")
    assert stat["num_episodes"] == meta["num_episodes"]
    L = meta["num_steps"]
    assert cpu(batch.valid)[:L, 0].all() and not cpu(batch.valid)[L:, 0].any()
    tr.optimizer.zero_grad(set_to_none=False)
    s = tr.compute_grad(batch)
    ret = torch.empty_like(batch.reward)
    from ic3net_b200 import _lib
    T = batch.reward.shape[0]
    _lib.check(_lib.load().ic3_returns_scan(T, 1, args.nagents, float(args.gamma), float(args.mean_ratio),
                                            batch.reward.data_ptr(), batch.episode_mask.data_ptr(),
                                            batch.episode_mini_mask.data_ptr(), ret.data_ptr(), _lib.stream()))
    assert np.allclose(cpu(ret)[:L, 0], z["returns"], rtol=1e-5, atol=1e-5)
    for q in ("action_loss", "value_loss", "entropy"):
        assert np.isclose(s[q], meta[q], rtol=2e-4, atol=1e-3), (q, s[q], meta[q])
    for key, prm in net.named_parameters():
        if "g_" + key in z.files:
            want = z["g_" + key]
            err = np.abs(cpu(prm.grad) - want).max() / max(np.abs(want).max(), 1e-30)
            assert err < 2e-3, (name, key, err)
        elif "gsample_" + key in z.files:
            got = cpu(prm.grad).astype(np.float64)
            want = z["gsum_" + key]
            assert np.isclose(got.sum(), want[0], rtol=2e-3, atol=2e-3 * want[1] / got.size * 50)
            gs = got.ravel()[::max(1, got.size // 2048)][:2048]
            ws = z["gsample_" + key]
            assert np.abs(gs - ws).max() <= 2e-3 * max(np.abs(ws).max(), 1e-30), (name, key)
