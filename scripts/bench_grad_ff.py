"""Cost of differentiating the non-recurrent tanh policies: device time, the rollout's share of it and peak memory of one
Trainer.train_batch with the non-recurrent gradient kernels (grad_impl 'kernels_ff') against the torch-autograd windowed
recompute (grad_impl 'autograd'), alternated in one process.  Runs: predator-prey hard (10 agents, dim 20, vision 1) with
8192 env slots at --batch_size 100 and 500 for models.MLP, the non-recurrent CommNet with 2 passes and the non-recurrent
IC3Net; traffic-junction hard with 4096 env slots, the non-recurrent IC3Net.

    python scripts/bench_grad_ff.py [--updates 2] [--rounds 1] [--batch_sizes 100,500] [--grad_window 10] [--only RUN]
                                    [--out FILE]

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


RUNS = {
    # name: (bench.py configuration, policy arguments, env slots)
    "pp_mlp": ("pp_hard_ic3net", dict(model="mlp", commnet=False, hard_attn=False, comm_passes=1), 8192),
    "pp_commnet_p2": ("pp_hard_ic3net", dict(model="commnet", commnet=True, hard_attn=False, comm_passes=2), 8192),
    "pp_ic3net": ("pp_hard_ic3net", dict(model="commnet", commnet=True, hard_attn=True, comm_passes=1), 8192),
    "tj_ic3net": ("tj_hard_ic3net", dict(model="commnet", commnet=True, hard_attn=True, comm_passes=1), 4096),
}


def build(run, grad_impl, batch_size, grad_window):
    import torch

    from bench import make_args
    from ic3net_b200 import data, models
    from ic3net_b200.action_utils import parse_action_args
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    conf, pol, slots = RUNS[run]
    pol = dict(pol)
    model = pol.pop("model")
    a = make_args(conf, 0, "index")
    for k, v in dict(pol, ic3net=False, recurrent=False, rnn_type="MLP", mean_ratio=1.0, policy_impl=None, nenvs=slots, record_for_grad=True,
                     batch_size=batch_size, grad_impl=grad_impl, batch_boundary="reference", value_coeff=0.01, entr=0.0,
                     gamma=1.0, normalize_rewards=False, detach_gap=10000, grad_window=grad_window,
                     share_weights=False, comm_mask_zero=False).items():
        setattr(a, k, v)
    env = data.init(a.env_name, a)
    a.num_inputs = env.observation_dim
    a.num_actions = [env.num_actions]
    a.dim_actions = 1
    if a.hard_attn and a.commnet:                       # the comm action head (main.py:134-140)
        a.num_actions, a.dim_actions = [env.num_actions, 2], 2
    parse_action_args(a)
    torch.manual_seed(0)
    net = (models.MLP if model == "mlp" else CommNetMLP)(a, a.num_inputs)
    tr = Trainer(a, net, env)
    assert tr.grad_ff == (grad_impl == "kernels_ff") and net.policy_impl == "simt"
    return tr


def measure(run, grad_impl, batch_size, opts):
    import torch

    from ic3net_b200.utils import merge_stat
    tr = build(run, grad_impl, batch_size, opts.grad_window)
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
    out = dict(run=run, grad_impl=grad_impl, env_slots=tr.env.env.nenvs, batch_size=batch_size, lock_steps=T,
               chunk_steps=getattr(tr, "ff_chunk_steps", None),
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
    ap.add_argument("--only", default=None, help="comma-separated subset of " + ",".join(RUNS))
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
    runs = opts.only.split(",") if opts.only else list(RUNS)
    for run in runs:
        # traffic junction: one batch size (its episodes are short and the slots halt together)
        for bs in (int(x) for x in opts.batch_sizes.split(",")[:1 if run.startswith("tj") else None]):
            for r in range(opts.rounds):
                for impl in ("kernels_ff", "autograd"):
                    emit(dict(round=r, **measure(run, impl, bs, opts)))
    emit(dict(card_after=card()))
    if opts.out:
        with open(opts.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
