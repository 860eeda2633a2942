"""Cost of one differentiable policy step at predator-prey hard (10 agents, dim 20, vision 1), IC3Net, 8192 env slots:

  module   forward + backward through CommNetMLP.forward with args.forward_grad = 'kernels' (ic3_policy_step +
           ic3_policy_step_backward), random upstream gradients of every output
  torch    the same step as fp32 torch autograd of trainer.policy_forward_torch (x from the env state by embedding_bag),
           the only other way to differentiate the module's step
  bptt     one ic3_bptt_step inside Trainer.compute_grad(grad_impl='kernels'): the slope of compute_grad's device time
           over rollouts of T1 and T2 lock-steps; the intercept is its per-call begin / finish cost (ic3_bptt_begin
           clears both operand-image sets)

    python scripts/bench_forward_grad.py [--iters 20] [--rounds 2] [--out FILE]

Device time by CUDA events around synchronised work; the three are alternated `rounds` times in one process.  Prints one
JSON line per measurement, and the card, its power limit and SM clock first and last."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def build(B):
    import torch

    from bench import make_args
    from ic3net_b200 import data
    from ic3net_b200.action_utils import parse_action_args
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    a = make_args("pp_hard_ic3net", 0, "index")
    for k, v in dict(nenvs=B, record_for_grad=True, grad_impl="kernels", value_coeff=0.01, entr=0.0, gamma=1.0,
                     mean_ratio=1.0, normalize_rewards=False, detach_gap=10000, obs_api="handle",
                     forward_grad="kernels", comm_passes=1, share_weights=False).items():
        setattr(a, k, v)
    env = data.init(a.env_name, a)
    a.num_inputs = env.observation_dim
    a.num_actions = [env.num_actions, 2]
    a.dim_actions = 2
    parse_action_args(a)
    torch.manual_seed(0)
    net = CommNetMLP(a, a.num_inputs)
    return Trainer(a, net, env)


def timed(fn, iters):
    import torch
    fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=20, help="timed steps per measurement")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--T", default="20,60", help="rollout lengths of the compute_grad slope")
    ap.add_argument("--out", default=None)
    opts = ap.parse_args()
    import torch
    import torch.nn.functional as F
    from bench_bptt_rnn import card
    from ic3net_b200.lazy_obs import LazyObs
    from ic3net_b200.trainer import policy_forward_torch
    torch.cuda.set_device(0)
    lines = [dict(card=card())]
    print(json.dumps(lines[0]), flush=True)

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    tr = build(opts.slots)
    net, e, args = tr.policy_net, tr.env.env, tr.args
    B, N, H = e.nenvs, args.nagents, args.hid_size
    R = B * N
    tr.rollout(8, 0)
    b = tr._buf
    h0, c0 = b["rec_h"][8].clone(), b["rec_c"][8].clone()
    info = dict(comm_action=b["comm"].clone(), alive_mask=b["alive"].clone())
    g = torch.Generator(device="cuda").manual_seed(0)
    up = [torch.randn(R, sum(args.naction_heads), device="cuda", generator=g), torch.randn(R, 1, device="cuda", generator=g),
          torch.randn(R, H, device="cuda", generator=g), torch.randn(R, H, device="cuda", generator=g)]
    shape = (B, N, tr.env.observation_dim)

    def module_step():
        h, c = h0.clone().requires_grad_(True), c0.clone().requires_grad_(True)
        action, value, (h2, c2) = net([LazyObs(e, shape), (h, c)], info)
        lp = torch.cat(action, -1).reshape(R, -1)
        ((lp * up[0]).sum() + (value * up[1]).sum() + (h2 * up[2]).sum() + (c2 * up[3]).sum()).backward()

    w = net._kernel_weights()

    def torch_step():
        h, c = h0.clone().requires_grad_(True), c0.clone().requires_grad_(True)
        idx, val = tr._pp_sparse_obs(e.loc)
        x = F.embedding_bag(idx, w["enc_w"].t(), per_sample_weights=val, mode="sum") + w["enc_b"]
        alive = info["alive_mask"].float()
        gate = alive * info["comm_action"].float()
        h2, c2, value, lps = policy_forward_torch(net, x, h, c, gate, alive.sum(1, keepdim=True))
        lp = torch.cat(lps, -1)
        ((lp * up[0]).sum() + (value * up[1]).sum() + (h2 * up[2]).sum() + (c2 * up[3]).sum()).backward()

    T1, T2 = (int(v) for v in opts.T.split(","))

    def compute_grad_ms(T):
        tr.rollout(T, 0)
        tr.optimizer.zero_grad(set_to_none=False)
        return timed(lambda: tr.compute_grad_device(None), 3)

    for r in range(opts.rounds):
        emit(dict(round=r, what="module forward + backward", slots=B, rows=R, ms_per_step=timed(module_step, opts.iters)))
        emit(dict(round=r, what="torch fp32 autograd of policy_forward_torch", slots=B, rows=R,
                  ms_per_step=timed(torch_step, opts.iters)))
        m1, m2 = compute_grad_ms(T1), compute_grad_ms(T2)
        slope = (m2 - m1) / (T2 - T1)
        emit(dict(round=r, what="compute_grad ic3_bptt_step", slots=B, rows=R, T=[T1, T2], compute_grad_ms=[m1, m2],
                  ms_per_bptt_step=slope, ms_per_call_overhead=m1 - slope * T1))
        # the rollout above left other records; re-take the module's state for the next round
        tr.rollout(8, 0)
        b = tr._buf
        h0.copy_(b["rec_h"][8])
        c0.copy_(b["rec_c"][8])
        info["comm_action"].copy_(b["comm"])
        info["alive_mask"].copy_(b["alive"])
    emit(dict(card_after=card()))
    if opts.out:
        with open(opts.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
