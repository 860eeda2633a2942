"""Traffic junction with the bool vocabulary against ``--vocab_type scalar``, alternated in one process: traffic-junction
hard (20 cars, dim 18, vision 0, 4096 env slots), IC3Net at hid_size 128 on the tensor-core policy step, index and dense
observations.

    python scripts/bench_tj_scalar.py [--updates 3] [--rounds 2] [--batch_size 100] [--nenvs 4096] [--out FILE]

Per measurement: the rollout's ms per lock-step and Trainer.train_batch ms per update (CUDA events around a synchronised
window).  grad_impl is 'auto': the bool vocabulary trains with the BPTT kernels, the scalar vocabulary -- which they do
not cover -- with the autograd recompute, so the train_batch numbers compare the two as a user gets them.  Prints one
JSON line per measurement, and the card, its power limit and SM clock first and last."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_bptt_rnn import card  # noqa: E402


def build(vocab_type, obs_mode, opts):
    import torch

    from bench import make_args
    from ic3net_b200 import data
    from ic3net_b200.action_utils import parse_action_args
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    a = make_args("tj_hard_ic3net", 0, obs_mode, nenvs=opts.nenvs)
    for k, v in dict(vocab_type=vocab_type, record_for_grad=True, batch_size=opts.batch_size, grad_impl="auto",
                     batch_boundary="reference", value_coeff=0.01, entr=0.0, gamma=1.0, normalize_rewards=False,
                     detach_gap=10000, policy_impl="tc").items():
        setattr(a, k, v)
    env = data.init(a.env_name, a)
    a.num_inputs = env.observation_dim
    a.num_actions, a.dim_actions = [env.num_actions, 2], 2          # IC3Net: env head + gating head
    parse_action_args(a)
    torch.manual_seed(0)
    net = CommNetMLP(a, a.num_inputs)
    return Trainer(a, net, env)


def measure(vocab_type, obs_mode, opts):
    import torch

    from ic3net_b200.utils import merge_stat
    tr = build(vocab_type, obs_mode, opts)
    T, _ = tr.batch_plan()
    tr.train_batch(0)                                   # warm-up: allocations, weight packing
    torch.cuda.synchronize()
    ms, roll = [], []
    for u in range(opts.updates):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        batch, stat = tr.run_batch(u + 1)               # = Trainer.train_batch, with an event after the rollout
        ev[1].record()
        tr.optimizer.zero_grad(set_to_none=False)
        s = tr.compute_grad(batch)
        merge_stat(s, stat)
        tr.optimizer.step(grad_div=stat["num_steps"])
        ev[2].record()
        torch.cuda.synchronize()
        ms.append(ev[0].elapsed_time(ev[2]))
        roll.append(ev[0].elapsed_time(ev[1]))
    out = dict(workload="tj_hard_ic3net", vocab_type=vocab_type, obs_mode=obs_mode, obs_dim=tr.env.observation_dim,
               env_slots=tr.env.env.nenvs, rows=tr.env.env.nenvs * tr.args.nagents, batch_size=opts.batch_size,
               lock_steps=T, grad_impl=tr.grad_impl, fused_encoder=tr.policy_net.fuses_encoder(tr.env.env),
               ms_per_update=ms, rollout_ms_per_lock_step=[r / T for r in roll])
    del tr
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=3, help="timed train_batch calls per measurement")
    ap.add_argument("--rounds", type=int, default=2, help="bool / scalar alternations per observation mode")
    ap.add_argument("--batch_size", type=int, default=100, help="--batch_size (lock-steps ~ this + max_steps)")
    ap.add_argument("--nenvs", type=int, default=4096, help="env slots")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    opts = ap.parse_args()
    import torch
    torch.set_num_threads(1)
    torch.cuda.set_device(0)
    lines = [dict(card=card())]

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    print(json.dumps(lines[0]), flush=True)
    for obs_mode in ("index", "dense"):
        for r in range(opts.rounds):
            for vocab_type in ("bool", "scalar"):
                emit(dict(round=r, **measure(vocab_type, obs_mode, opts)))
    emit(dict(card_after=card()))
    if opts.out:
        with open(opts.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
