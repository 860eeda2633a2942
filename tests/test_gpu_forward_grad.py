"""CommNetMLP.forward with args.forward_grad = 'kernels': a differentiable policy step whose backward is
ic3_policy_step_backward (csrc/bptt_tc.cu, the BPTT kernels with the heads in their upstream-gradient form).

Covered:
  - one step under random upstream gradients (d log-probs, d value, d h', d c') against torch float64 autograd of the
    same step on float64 copies of the parameters, x rebuilt from the env state, at full batch size (predator-prey hard
    with 8192 slots, traffic junction hard with 4096 slots, states with episode starts and dead cars) and on ragged
    tiles: 1, 2 and 4 comm passes, share_weights, hard attention, comm_mode sum, comm_mask_zero, --enemy_comm, and the
    IC / IRIC tanh RNN on 'simt' and 'tc_tanh';
  - a T-step chain through forward with the reference's loss (trainer.py:160-220 on the returned tensors), the caller's
    detach_gap detaches and loss.backward(), against Trainer.compute_grad(grad_impl='kernels') on the same trajectory;
  - outputs bit-identical with and without the opt-in and under no_grad, no grad_fn without the opt-in, gradients
    bit-identical run to run;
  - the refusals, and the RuntimeError when the weights change between forward and backward.

Bar (that of the BPTT tests): per tensor max |kernels - float64| <= 1e-4 of the float64 tensor's largest entry; the
encoder weight also per input column; the action heads' entries also 2^-20 of their sum of |terms|."""
import pytest
import torch

from bptt_ref import heads_abs_sums, returns_and_advantages
from gpu_harness import OPT_IN, assert_within_bar as within_bar, handle, one_step, passes_trainer, rnn_trainer, set_state


def lstm_trainer(name, B, passes, share, **over):
    return passes_trainer(name, B, comm_passes=passes, share_weights=share, **over)


LSTM_STEP = [
    ("grad_pp_hard_ic3net_h128", 8192, 1, False, {}),
    ("grad_pp_hard_ic3net_h128", 8192, 2, False, {}),
    ("grad_pp_hard_ic3net_h128", 1000, 4, True, {}),
    ("grad_tj_hard_ic3net_h128", 4096, 1, False, {}),
    ("grad_tj_hard_ic3net_h128", 333, 3, True, dict(comm_mode="sum", hard_attn=False)),
    ("grad_tj_medium_v1_ic_h128", 700, 1, False, {}),                  # comm_mask_zero, vision 1
    ("grad_pp_enemy_ic3net_h128", 517, 2, False, {}),                  # --enemy_comm
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,passes,share,over", LSTM_STEP)
def test_one_step_matches_float64(name, B, passes, share, over):
    tr = lstm_trainer(name, B, passes, share, seed=5, id0=0, **dict(OPT_IN, **over))
    tr.rollout(tr.args.max_steps + 4, 0)
    b = tr._buf
    assert int(b["s_fresh"][1:].sum()) > 0                             # episode starts inside the rollout
    t = tr.args.max_steps - 2                                          # mid-episode
    if tr.is_tj:                                                       # live and dead cars in the differentiated state
        assert 0 < int(b["s_tjalive"][t].sum()) < b["s_tjalive"][t].numel()
    got, ref, sums = one_step(tr, t)
    within_bar(got, ref, sums, "%s B=%d passes=%d share=%s %s" % (name, B, passes, share, over))


@pytest.mark.gpu
@pytest.mark.parametrize("name,B", [("gradrnn_pp_hard_ic", 8192), ("gradrnn_tj_iric", 901)])
@pytest.mark.parametrize("impl", ["simt", "tc_tanh"])
def test_one_step_tanh_rnn_matches_float64(name, B, impl):
    tr = rnn_trainer(name, B, seed=5, id0=0, policy_impl=impl, **OPT_IN)
    tr.rollout(tr.args.max_steps + 4, 0)
    got, ref, sums = one_step(tr, tr.args.max_steps - 2)
    within_bar(got, ref, sums, "%s B=%d %s" % (name, B, impl))


# ---------------------------------------------------------------------------------------------------- through time

def chain_grads(tr):
    """The recorded trajectory re-run through forward with the reference's loss (trainer.py:160-220 on the returned
    tensors, the caller's detaches of trainer.py:56-60) and loss.backward(): {name: grad}."""
    net, args, e, b = tr.policy_net, tr.args, tr.env.env, tr._buf
    T, B, N, H = b["T"], e.nenvs, args.nagents, args.hid_size
    lstm = net._cfg_proto["cell"] == 0
    hard = bool(args.hard_attn) and bool(args.commnet)
    ret, adv = returns_and_advantages(tr)
    ret, adv = ret.reshape(T, B, N), adv.reshape(T, B, N)
    net.zero_grad(set_to_none=True)
    h = torch.zeros(B * N, H, device="cuda")
    c = torch.zeros(B * N, H, device="cuda")
    loss = 0.0
    for t in range(T):
        set_state(tr, t)
        fresh = b["s_fresh"][t].bool()
        keep = (~fresh).float().repeat_interleave(N).unsqueeze(1)
        h, c = h * keep, c * keep                                             # trainer.py:45-51
        f2 = fresh.unsqueeze(1)
        info = dict(alive_mask=torch.where(f2, torch.ones_like(b["s_alive"][t]), b["s_alive"][t]))
        if hard:
            info["comm_action"] = torch.where(f2, torch.zeros_like(b["s_comm"][t]), b["s_comm"][t])
        action, value, hid = net([handle(tr), (h, c) if lstm else h], info)
        h, c = hid if lstm else (hid, c)
        act = b["action"][t].long()
        alive_post = b["ralive"][t].float()
        vmask = b["valid"][t].float().view(B, 1, 1)
        lp_taken = torch.zeros(B, N, device="cuda")
        ent = 0.0
        for k, lp in enumerate(action):
            lp_taken = lp_taken + lp.gather(-1, act[..., k:k + 1]).squeeze(-1)        # utils.py:42-46
            ent = ent - (lp * lp.exp() * vmask).sum()
        loss = loss + (-adv[t] * lp_taken * alive_post).sum()                          # trainer.py:198-201
        loss = loss + args.value_coeff * ((value.view(B, N) - ret[t]).pow(2) * alive_post).sum()
        if args.entr > 0:
            loss = loss - args.entr * ent
        if args.detach_gap <= args.max_steps:                                         # trainer.py:56-60
            cut = (((b["s_tep"][t] + 1) % args.detach_gap) == 0).repeat_interleave(N).unsqueeze(1)
            h = torch.where(cut, h.detach(), h)
            c = torch.where(cut, c.detach(), c)
    loss.backward()
    return {n: p.grad.detach().double().clone() for n, p in net.named_parameters() if p.grad is not None}


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,passes,share,T", [("grad_pp_hard_ic3net_h128", 300, 1, False, 24),
                                                   ("grad_tj_hard_ic3net_h128", 130, 2, True, 29),
                                                   ("gradrnn_pp_ic_detach", 200, 1, False, 13)])
def test_chain_matches_compute_grad(name, B, passes, share, T):
    if name.startswith("gradrnn"):
        tr = rnn_trainer(name, B, seed=9, id0=3, **OPT_IN)
    else:
        tr = lstm_trainer(name, B, passes, share, seed=9, id0=3, **OPT_IN)
    tr.rollout(T, 0)
    b, args = tr._buf, tr.args
    assert int(b["s_fresh"][1:].sum()) > 0 and int((((b["s_tep"] + 1) % args.detach_gap) == 0).sum()) > 0
    tr.optimizer.zero_grad(set_to_none=False)
    tr.compute_grad(None)
    want = {n: p.grad.detach().double().clone() for n, p in tr.policy_net.named_parameters()}
    got = chain_grads(tr)
    want = {k: v for k, v in want.items() if k in got or float(v.abs().max()) != 0.0}
    assert set(want) <= set(got), set(want) - set(got)
    within_bar(got, want, heads_abs_sums(tr), "%s chain T=%d vs compute_grad" % (name, T))


# ---------------------------------------------------------------------------------------------------- unchanged

@pytest.mark.gpu
def test_outputs_bit_identical_and_gradients_deterministic():
    tr = lstm_trainer("grad_pp_hard_ic3net_h128", 200, 2, False, **OPT_IN)
    tr.rollout(6, 0)
    net, b = tr.policy_net, tr._buf
    T = b["T"]
    info = dict(comm_action=b["comm"], alive_mask=b["alive"])
    hc = (b["rec_h"][T], b["rec_c"][T])
    outs = []
    with torch.no_grad():
        outs.append(net([handle(tr), hc], info))
    net.forward_grad = None
    outs.append(net([handle(tr), hc], info))
    assert outs[-1][1].grad_fn is None and outs[-1][2][0].grad_fn is None
    net.forward_grad = "kernels"
    outs.append(net([handle(tr), hc], info))
    assert outs[-1][1].grad_fn is not None
    flat = [torch.cat([torch.cat(a, -1).reshape(-1), v.reshape(-1), hid[0].reshape(-1), hid[1].reshape(-1)])
            for a, v, hid in outs]
    assert all(torch.equal(flat[0], f) for f in flat[1:])
    grads = []
    for _ in range(2):
        got, _, _ = one_step(tr, 4, seed=3)
        grads.append(got)
    assert all(torch.equal(grads[0][k], grads[1][k]) for k in grads[0])


# ---------------------------------------------------------------------------------------------------- refusals

@pytest.mark.gpu
def test_refusals():
    from ic3net_b200 import models
    from ic3net_b200.comm import CommNetMLP
    tr = lstm_trainer("grad_pp_hard_ic3net_h128", 8, 1, False, **OPT_IN)
    args = tr.args
    a = lambda **kw: type(args)(**dict(vars(args), **kw))
    for bad in (dict(recurrent=False, policy_impl="simt"), dict(recurrent=False, policy_impl="tc_ff"),
                dict(policy_impl="simt"), dict(hid_size=64, policy_impl="simt")):
        with pytest.raises(NotImplementedError):
            CommNetMLP(a(**bad), args.num_inputs)
    with pytest.raises(NotImplementedError):
        models.MLP(a(), args.num_inputs)
    with pytest.raises(ValueError):
        CommNetMLP(a(forward_grad="autograd"), args.num_inputs)
    # a dense observation tensor with grad enabled
    net = tr.policy_net
    tr.rollout(2, 0)
    b = tr._buf
    info = dict(comm_action=b["comm"], alive_mask=b["alive"])
    hc = (b["rec_h"][2], b["rec_c"][2])
    with pytest.raises(NotImplementedError, match="obs_api='handle'"):
        net([handle(tr).dense(), hc], info)
    with torch.no_grad():                                     # inference is unchanged
        net([handle(tr).dense(), hc], info)
    # weights changed between forward and backward
    _, value, _ = net([handle(tr), hc], info)
    with torch.no_grad():
        net.value_head.bias.add_(1.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        value.sum().backward()
    # environments outside the kernels: a vision window wider than 5 x 5, the scalar vocabulary
    for name, over in (("grad_pp_hard_ic3net_h128", dict(vision=3)), ("grad_tj_hard_ic3net_h128", dict(vocab_type="scalar"))):
        t2 = lstm_trainer(name, 8, 1, False, grad_impl="auto", **dict(OPT_IN, **over))
        t2.rollout(2, 0)
        b2 = t2._buf
        with pytest.raises(NotImplementedError):
            t2.policy_net([handle(t2), (b2["rec_h"][2] if "rec_h" in b2 else b2["h"], b2["c"])],
                          dict(comm_action=b2["comm"], alive_mask=b2["alive"]))
