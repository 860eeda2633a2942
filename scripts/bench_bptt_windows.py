"""Cost of the BPTT kernels' windowed (h, c) records: device time and peak memory of Trainer.train_batch at predator-prey
hard, 8192 env slots (bench.py's train_batch leg settings), with full records against forced windows at --batch_size
500 (alternated, in one process), and with windows at batch sizes whose full records do not fit on an 80 GB card.

    python scripts/bench_bptt_windows.py [--updates 2] [--rounds 3] [--out FILE]

Prints one JSON line per measurement (and the card, its power limit and SM clock first)."""
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


def build(batch_size, windows):
    import torch

    from bench import make_args
    from ic3net_b200 import data
    from ic3net_b200.action_utils import parse_action_args
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    a = make_args("pp_hard_ic3net", 0, "index")
    a.policy_impl = "tc"
    for k, v in dict(record_for_grad=True, batch_size=batch_size, grad_impl="kernels", batch_boundary="reference",
                     value_coeff=0.01, entr=0.0, gamma=1.0, normalize_rewards=False, detach_gap=10000,
                     grad_window=40).items():
        setattr(a, k, v)
    env = data.init(a.env_name, a)
    a.num_inputs = env.observation_dim
    a.num_actions = [env.num_actions] + ([2] if a.hard_attn else [])
    a.dim_actions = len(a.num_actions)
    parse_action_args(a)
    torch.manual_seed(0)
    net = CommNetMLP(a, a.num_inputs)
    tr = Trainer(a, net, env)
    if windows:
        tr.RECORD_BYTES_LIMIT = 0
    return tr


def measure(batch_size, windows, updates):
    import torch
    tr = build(batch_size, windows)
    T, _ = tr.batch_plan()
    tr.train_batch(0)                                   # warm-up: allocations, weight packing
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms, steps = [], 0
    for u in range(updates):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        stat = tr.train_batch(u + 1)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
        steps += int(stat["num_steps"])
    out = dict(batch_size=batch_size, lock_steps=T, record_mode=tr.record_mode,
               record_gb=tr._record_bytes(T)[tr.record_mode] / 1e9, full_record_gb=tr._record_bytes(T)["full"] / 1e9,
               ms_per_update=ms, ms_per_lock_step=[m / T for m in ms],
               agent_env_steps_per_s=steps * tr.args.nagents / (sum(ms) * 1e-3),
               peak_allocated_gb=torch.cuda.max_memory_allocated() / 1e9)
    del tr
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=2, help="timed train_batch calls per measurement")
    ap.add_argument("--rounds", type=int, default=3, help="full / window alternations at batch 500")
    ap.add_argument("--large", default="1000,1500", help="batch sizes measured with windows only")
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
    for r in range(opts.rounds):
        for windows in (False, True):
            emit(dict(round=r, **measure(500, windows, opts.updates)))
    for bs in [int(x) for x in opts.large.split(",") if x]:
        emit(measure(bs, False, opts.updates))           # default selection: windows where full records do not fit
    emit(dict(card_after=card()))
    if opts.out:
        with open(opts.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
