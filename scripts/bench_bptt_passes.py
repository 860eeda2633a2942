"""Cost of differentiating comm_passes > 1 / share_weights policies: device time and peak memory of Trainer.train_batch
at predator-prey hard, 8192 env slots, with the BPTT kernels (grad_impl 'kernels') against the torch-autograd windowed
recompute (grad_impl 'autograd'), alternated in one process, for comm_passes 2 and 4 and comm_passes 3 with
share_weights (and comm_passes 1 for reference).

    python scripts/bench_bptt_passes.py [--updates 2] [--rounds 2] [--batch_size 100] [--grad_window 10] [--out FILE]

Prints one JSON line per measurement (and the card, its power limit and SM clock first and last).  Each line names
its stream schedule: IC3_BPTT_OVERLAP=0 (read once per process) keeps every BPTT kernel on the caller's stream, so
the two schedules are compared by alternating runs of the script with --kernels_only, with and without it."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [(1, False), (2, False), (4, False), (3, True)]     # (comm_passes, share_weights)


def card():
    import torch
    q = "name,power.limit,power.max_limit,clocks.sm,clocks.max.sm,temperature.gpu"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=" + q,
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi unavailable: %s" % e
    return dict(device=torch.cuda.get_device_name(), nvidia_smi_fields=q, nvidia_smi=out)


def build(passes, share, grad_impl, batch_size, grad_window):
    import torch

    from bench import make_args
    from ic3net_b200 import data
    from ic3net_b200.action_utils import parse_action_args
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    a = make_args("pp_hard_ic3net", 0, "index")
    a.policy_impl = "tc"
    for k, v in dict(record_for_grad=True, batch_size=batch_size, grad_impl=grad_impl, batch_boundary="reference",
                     value_coeff=0.01, entr=0.0, gamma=1.0, normalize_rewards=False, detach_gap=10000,
                     grad_window=grad_window, comm_passes=passes, share_weights=share).items():
        setattr(a, k, v)
    env = data.init(a.env_name, a)
    a.num_inputs = env.observation_dim
    a.num_actions = [env.num_actions] + ([2] if a.hard_attn else [])
    a.dim_actions = len(a.num_actions)
    parse_action_args(a)
    torch.manual_seed(0)
    net = CommNetMLP(a, a.num_inputs)
    tr = Trainer(a, net, env)
    assert tr.grad_kernels == (grad_impl == "kernels")
    return tr


def measure(passes, share, grad_impl, opts):
    import torch
    tr = build(passes, share, grad_impl, opts.batch_size, opts.grad_window)
    T, _ = tr.batch_plan()
    tr.train_batch(0)                                   # warm-up: allocations, weight packing
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms, steps = [], 0
    for u in range(opts.updates):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        stat = tr.train_batch(u + 1)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
        steps += int(stat["num_steps"])
    ws = int(tr._bptt["ws"].numel()) if tr._bptt is not None else 0
    overlap = os.environ.get("IC3_BPTT_OVERLAP")
    out = dict(schedule="one-stream" if overlap is not None and int(overlap) == 0 else "two-stream", comm_passes=passes, share_weights=share, grad_impl=grad_impl, env_slots=tr.env.env.nenvs,
               batch_size=opts.batch_size, lock_steps=T, record_mode=tr.record_mode,
               grad_window=opts.grad_window if grad_impl == "autograd" else None,
               bptt_workspace_gb=ws / 1e9, ms_per_update=ms,
               agent_env_steps_per_s=steps * tr.args.nagents / (sum(ms) * 1e-3),
               peak_allocated_gb=torch.cuda.max_memory_allocated() / 1e9)
    del tr
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=2, help="timed train_batch calls per measurement")
    ap.add_argument("--rounds", type=int, default=2, help="kernels / autograd alternations per case")
    ap.add_argument("--batch_size", type=int, default=100, help="--batch_size of the update (lock-steps ~ this + max_steps)")
    ap.add_argument("--grad_window", type=int, default=10, help="steps per autograd recompute window")
    ap.add_argument("--kernels_only", action="store_true", help="skip the autograd runs")
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
    for passes, share in CASES:
        for r in range(opts.rounds):
            for impl in ("kernels",) if opts.kernels_only else ("kernels", "autograd"):
                emit(dict(round=r, **measure(passes, share, impl, opts)))
    emit(dict(card_after=card()))
    if opts.out:
        with open(opts.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
