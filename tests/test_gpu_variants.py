"""SURVEY 8(f)-4: the other policy variants of the reference on the CUDA kernels -- `comm_passes > 1`, `share_weights`,
the non-recurrent tanh branch of CommNetMLP (comm.py:63-70,127-131,220-224) and the independent-controller baselines
of models.py (MLP, RNN with the tanh or the LSTM recurrence) -- against forward fixtures produced by the UNMODIFIED
reference modules (tests/golden/var_*.npz: their own seeded state_dict, inputs, outputs)."""
import argparse

import numpy as np
import pytest
import torch

from gpu_harness import close, variant_net
from helpers import golden_names, load_golden

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("impl", [None, "simt"])
@pytest.mark.parametrize("name", golden_names("var_"))
def test_variant_forward_matches_reference(name, impl):
    """impl None = the implementation the module picks (wgmma for the LSTM-cell variants at hid_size 128, whatever the
    number of comm passes); 'simt' = the fp32 kernel forced on those same cases."""
    meta, z = load_golden(name)
    a, net = variant_net(meta, z, impl)
    if impl == "simt" and not (net.tc_capable and a.hid_size == 128):
        pytest.skip("the module picks the SIMT kernel for this case anyway")
    n, H = a.nagents, a.hid_size
    nrep = z["obs"].shape[0]
    B = nrep                                              # all fixture cases as ONE batch of independent envs
    obs = torch.tensor(z["obs"], dtype=torch.float32, device="cuda")
    info = {}
    if meta["hard_attn"]:
        info["comm_action"] = torch.tensor(z["comm"], dtype=torch.uint8, device="cuda")
    if meta["use_alive"]:
        info["alive_mask"] = torch.tensor(z["alive"], dtype=torch.uint8, device="cuda")
    h = torch.tensor(z["h"], dtype=torch.float32, device="cuda").reshape(B * n, H)
    c = torch.tensor(z["c"], dtype=torch.float32, device="cuda").reshape(B * n, H)
    if not meta["carries"]:
        act, val = net(obs, info)
        h2 = c2 = None
    elif meta["lstm"]:
        act, val, (h2, c2) = net([obs, (h, c)], info)
    else:
        act, val, h2 = net([obs, h], info)
        c2 = None
    torch.cuda.synchronize()
    assert close(val.reshape(B, n).cpu().numpy(), z["value"]), name
    for k in range(len(meta["heads"])):
        assert close(act[k].cpu().numpy(), z["logp%d" % k]), (name, k)
    if h2 is not None:
        assert close(h2.reshape(B, n, H).cpu().numpy(), z["h2"]), name
    if c2 is not None:
        assert close(c2.reshape(B, n, H).cpu().numpy(), z["c2"]), name
    expect_tc = impl is None and bool(meta["lstm"]) and H == 128        # LSTM cell on the encoded observation
    assert (net.policy_impl == "tc") == expect_tc
    if expect_tc:
        net.check_errors()                                               # pipeline watchdog / fp16 range flags


def test_tanh_cell_variant_on_tensor_core_path_is_refused():
    for name in ("var_commnet_nonrec2", "var_mlp", "var_rnn_tanh"):
        meta, z = load_golden(name)
        with pytest.raises(NotImplementedError):
            variant_net(meta, z, policy_impl="tc")


@pytest.mark.parametrize("model,extra", [("rnn", dict(rnn_type="MLP")), ("rnn", dict(rnn_type="LSTM")), ("mlp", {}),
                                         ("commnet", dict(comm_passes=2, share_weights=True)),
                                         ("commnet", dict(comm_passes=3, hard_attn=False)),
                                         ("commnet", dict(comm_passes=2, share_weights=True, policy_impl="simt")),
                                         ("commnet", dict(recurrent=False, comm_passes=2))])
def test_variant_trains_and_recompute_agrees_with_the_kernels(model, extra):
    """A full update (rollout kernels -> compute_grad -> RMSprop) for every family, and the differentiable recompute
    that produces the gradient must reproduce the values / log-probs the rollout kernels recorded."""
    from ic3net_b200 import data, models
    from ic3net_b200.action_utils import parse_action_args
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer, policy_forward_torch
    a = argparse.Namespace(env_name="predator_prey", nagents=3, nfriendly=3, dim=5, vision=1, mode="mixed", nenemies=1,
                           no_stay=False, moving_prey=False, enemy_comm=False, nenvs=6, seed=5, env_id0=0,
                           hid_size=128, recurrent=(model != "mlp"), rnn_type="LSTM", commnet=(model == "commnet"),
                           hard_attn=(model == "commnet"), comm_action_one=False, comm_mode="avg", comm_passes=1,
                           comm_mask_zero=False, comm_init="uniform", share_weights=False, max_steps=10,
                           batch_size=20, lrate=1e-3, obs_mode="index", use_graph=False, continuous=False,
                           detach_gap=4, gamma=0.9, mean_ratio=0.5, value_coeff=0.01, entr=0.01,
                           normalize_rewards=False, record_for_grad=True, grad_window=8)
    for k, v in extra.items():
        setattr(a, k, v)
    env = data.init(a.env_name, a)
    a.num_inputs = env.observation_dim
    a.num_actions = [env.num_actions] + ([2] if a.hard_attn else [])
    a.dim_actions = len(a.num_actions)
    parse_action_args(a)
    torch.manual_seed(3)
    net = {"commnet": CommNetMLP, "mlp": models.MLP, "rnn": models.RNN}[model](a, a.num_inputs)
    tr = Trainer(a, net, env)
    before = tr.optimizer.flat_params.clone()
    stat = tr.train_batch(0)
    assert np.isfinite(stat["action_loss"]) and np.isfinite(stat["value_loss"]) and stat["num_steps"] >= 6 * 20
    assert not torch.equal(before, tr.optimizer.flat_params)
    # recompute of the recorded rollout vs what the kernels wrote (new rollout with the updated weights)
    batch, stat = tr.run_batch(1)
    b = tr._buf
    B, N, H = 6, 3, 128
    T = b["T"]
    with torch.no_grad():
        h = torch.zeros(B * N, H, device="cuda")
        c = torch.zeros(B * N, H, device="cuda")
        w = net._kernel_weights()
        worst = 0.0
        for t in range(T):
            keep = (1 - b["s_fresh"][t].float()).repeat_interleave(N).unsqueeze(1)
            h, c = h * keep, c * keep
            idx, val = tr._pp_sparse_obs(b["s_loc"][t])
            x = torch.nn.functional.embedding_bag(idx, w["enc_w"].t().contiguous(), per_sample_weights=val, mode="sum") + w["enc_b"]
            fresh = b["s_fresh"][t].bool().unsqueeze(1)
            alive = torch.ones(B, N, device="cuda")
            g = alive
            if a.hard_attn and a.commnet:
                g = g * torch.where(fresh, torch.zeros_like(b["s_comm"][t]), b["s_comm"][t]).float()
            h, c, value, logps = policy_forward_torch(net, x, h, c, g, alive.sum(1, keepdim=True))
            v = (b["valid"][t] != 0)
            if not bool(v.any()):
                continue
            got_v = b["value"][t].view(B, N)[v]
            worst = max(worst, float((got_v - value.view(B, N)[v]).abs().max()))
            lp = torch.cat(logps, -1).view(B, N, -1)[v]
            worst = max(worst, float((b["logp"][t][v] - lp).abs().max()))
    assert worst < 2e-4, worst
