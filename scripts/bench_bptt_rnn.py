"""Cost of differentiating the IC baseline (models.RNN with the tanh recurrence, rnn_type 'MLP', on the SIMT policy
kernel): device time, the rollout's share of it and peak memory of one Trainer.train_batch at predator-prey hard
(10 agents, dim 20, vision 1), 8192 env slots, with the BPTT kernels (grad_impl 'kernels') against the torch-autograd
windowed recompute (grad_impl 'autograd'), alternated in one process, at --batch_size 100 and 500.

    python scripts/bench_bptt_rnn.py [--updates 2] [--rounds 1] [--batch_sizes 100,500] [--grad_window 10] [--out FILE]

Prints one JSON line per measurement, and the card, its power limit and SM clock first and last.  The rollout (SIMT
forward, env step) is the same for both: its share is timed with CUDA events around run_batch."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    q = "name,power.limit,power.max_limit,clocks.sm,clocks.max.sm,temperature.gpu"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=" + q,
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi unavailable: %s" % e
    return dict(device=torch.cuda.get_device_name(), nvidia_smi_fields=q, nvidia_smi=out)


def build(grad_impl, batch_size, grad_window):
    import torch

    from bench import make_args
    from ic3net_b200 import data, models
    from ic3net_b200.action_utils import parse_action_args
    from ic3net_b200.trainer import Trainer
    a = make_args("pp_hard_ic3net", 0, "index")
    # IC: --recurrent without --commnet (models.RNN, rnn_type 'MLP'), no hard attention
    for k, v in dict(commnet=False, recurrent=True, rnn_type="MLP", hard_attn=False, mean_ratio=1.0, policy_impl=None,
                     record_for_grad=True, batch_size=batch_size, grad_impl=grad_impl, batch_boundary="reference",
                     value_coeff=0.01, entr=0.0, gamma=1.0, normalize_rewards=False, detach_gap=10000,
                     grad_window=grad_window, comm_passes=1, share_weights=False).items():
        setattr(a, k, v)
    env = data.init(a.env_name, a)
    a.num_inputs = env.observation_dim
    a.num_actions = [env.num_actions]
    a.dim_actions = 1
    parse_action_args(a)
    torch.manual_seed(0)
    net = models.RNN(a, a.num_inputs)
    tr = Trainer(a, net, env)
    assert tr.grad_kernels == (grad_impl == "kernels") and net.policy_impl == "simt"
    return tr


def measure(grad_impl, batch_size, opts):
    import torch

    from ic3net_b200.utils import merge_stat
    tr = build(grad_impl, batch_size, opts.grad_window)
    T, _ = tr.batch_plan()
    tr.train_batch(0)                                   # warm-up: allocations, weight packing
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms, roll, steps = [], [], 0
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
        steps += int(stat["num_steps"])
    out = dict(policy="IC (models.RNN, tanh)", grad_impl=grad_impl, env_slots=tr.env.env.nenvs, batch_size=batch_size,
               lock_steps=T, record_mode=tr.record_mode,
               grad_window=opts.grad_window if grad_impl == "autograd" else None,
               ms_per_update=ms, rollout_ms=roll, rollout_share=[r / m for r, m in zip(roll, ms)],
               agent_env_steps_per_s=steps * tr.args.nagents / (sum(ms) * 1e-3),
               peak_allocated_gb=torch.cuda.max_memory_allocated() / 1e9)
    del tr
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=2, help="timed train_batch calls per measurement")
    ap.add_argument("--rounds", type=int, default=1, help="kernels / autograd alternations per batch size")
    ap.add_argument("--batch_sizes", default="100,500", help="--batch_size values (lock-steps ~ this + max_steps)")
    ap.add_argument("--grad_window", type=int, default=10, help="steps per autograd recompute window")
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
    for bs in (int(x) for x in opts.batch_sizes.split(",")):
        for r in range(opts.rounds):
            for impl in ("kernels", "autograd"):
                emit(dict(round=r, **measure(impl, bs, opts)))
    emit(dict(card_after=card()))
    if opts.out:
        with open(opts.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
