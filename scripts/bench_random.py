"""Rollout rate of the Random baseline (--random, models.Random: ic3_random_policy_step + the env step per lock-step):
Trainer.run_batch timed with CUDA events at predator-prey hard (10 agents, dim 20, vision 1, 80 steps, 8192 env slots)
and traffic-junction hard (20 agents, dim 18, 80 steps, 4096 env slots), eager and as a CUDA graph.

    python scripts/bench_random.py [--updates 5] [--batch_size 500] [--out FILE]

Prints one JSON line per measurement (agent-env-steps/s = real steps x agents / device time of run_batch, which
includes its one device->host copy of the statistics), and the card, its power limit and SM clock first and last."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_bptt_rnn import card  # noqa: E402


def build(wl, batch_size, use_graph):
    import torch

    from bench import make_args
    from ic3net_b200 import data, models
    from ic3net_b200.action_utils import parse_action_args
    from ic3net_b200.trainer import Trainer
    a = make_args(wl, 0, "index")
    for k, v in dict(commnet=False, recurrent=False, random=True, hard_attn=False, comm_action_one=False,
                     mean_ratio=1.0, batch_size=batch_size, batch_boundary="reference", use_graph=use_graph).items():
        setattr(a, k, v)
    env = data.init(a.env_name, a)
    a.num_inputs = env.observation_dim
    a.num_actions = [env.num_actions]
    a.dim_actions = 1
    parse_action_args(a)
    torch.manual_seed(0)
    return Trainer(a, models.Random(a, a.num_inputs), env)


def measure(wl, batch_size, use_graph, updates):
    import torch
    tr = build(wl, batch_size, use_graph)
    T, _ = tr.batch_plan()
    tr.run_batch(0)                                      # warm-up: allocations, graph capture
    torch.cuda.synchronize()
    ms, steps = [], 0
    for u in range(updates):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        _, stat = tr.run_batch(u + 1)
        ev[1].record()
        torch.cuda.synchronize()
        ms.append(ev[0].elapsed_time(ev[1]))
        steps += int(stat["num_steps"])
    out = dict(policy="Random (models.Random)", workload=wl, use_graph=use_graph, env_slots=tr.env.env.nenvs,
               agents=tr.args.nagents, batch_size=batch_size, lock_steps=T, ms_per_run_batch=ms,
               agent_env_steps_per_s=steps * tr.args.nagents / (sum(ms) * 1e-3))
    del tr
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=5, help="timed run_batch calls per measurement")
    ap.add_argument("--batch_size", type=int, default=500, help="--batch_size (steps per env slot and batch)")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    opts = ap.parse_args()
    import torch
    torch.set_num_threads(1)
    torch.cuda.set_device(0)
    lines = []

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    emit(dict(card=card()))
    for wl in ("pp_hard_ic3net", "tj_hard_ic3net"):
        for use_graph in (False, True):
            emit(measure(wl, opts.batch_size, use_graph, opts.updates))
    emit(dict(card_after=card()))
    if opts.out:
        with open(opts.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
