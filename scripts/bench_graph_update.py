"""Trainer.train_batch milliseconds per update, eager and with graph_update, alternated update by update on one Trainer
in one process, at --batch_size 500 (the reference's update: 16 workers x 500 steps is --nenvs 16 here).

    python scripts/bench_graph_update.py [--updates 3] [--only NAME[,NAME]] [--out FILE]

Setups: predator-prey hard IC3Net (LSTM on the tensor cores, BPTT kernels) at 16, 128, 1024 and 8192 env slots;
traffic-junction hard IC3Net at 16, 128 and 4096; IC (tanh RNN, policy_impl tc_tanh) and models.MLP (tc_ff + kernels_ff)
at 16.  Each update is timed by the host clock from the call to a device synchronise after it.  The first update of
each mode (and the capture of graph_update) is warm-up and not timed.  Prints one JSON line per setup, and the card,
its power limit and SM clock first and last."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PP = ["--env_name", "predator_prey", "--nagents", "10", "--dim", "20", "--vision", "1", "--max_steps", "80",
      "--mode", "mixed", "--nenemies", "1", "--hid_size", "128", "--detach_gap", "10"]
TJ = ["--env_name", "traffic_junction", "--nagents", "20", "--dim", "18", "--vision", "0", "--max_steps", "80",
      "--difficulty", "hard", "--add_rate_min", "0.05", "--add_rate_max", "0.05", "--hid_size", "128",
      "--detach_gap", "10"]
IC3NET = ["--ic3net", "--recurrent"]
SETUPS = [("pp_ic3net", PP + IC3NET, n) for n in (16, 128, 1024, 8192)] + \
         [("tj_ic3net", TJ + IC3NET, n) for n in (16, 128, 4096)] + \
         [("pp_ic_tc_tanh", PP + ["--recurrent", "--policy_impl", "tc_tanh"], 16),
          ("pp_mlp_tc_ff", PP + ["--policy_impl", "tc_ff", "--grad_impl", "kernels_ff"], 16)]


def card():
    import torch
    q = "name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=" + q,
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi unavailable: %s" % e
    return dict(device=torch.cuda.get_device_name(), nvidia_smi_fields=q, nvidia_smi=out)


def make_trainer(argv):
    """The Trainer ic3net_b200.main builds for these flags (one process, seed 1)."""
    import torch
    from ic3net_b200 import data, main as m
    from ic3net_b200.action_utils import parse_action_args
    from ic3net_b200.trainer import Trainer
    from ic3net_b200.utils import init_args_for_env
    parser = m.build_parser()
    init_args_for_env(parser, ['x'] + list(argv))
    args = m.derive_args(parser.parse_args(argv))
    args.env_id0 = 0
    torch.manual_seed(args.seed)
    env = data.init(args.env_name, args, False)
    args.num_actions = env.num_actions if isinstance(env.num_actions, (list, tuple)) else [env.num_actions]
    args.dim_actions = env.dim_actions
    args.num_inputs = env.observation_dim
    if args.hard_attn and args.commnet:
        args.num_actions = [*args.num_actions, 2]
        args.dim_actions = env.dim_actions + 1
    if args.commnet and (args.recurrent or args.rnn_type == 'LSTM'):
        args.recurrent, args.rnn_type = True, 'LSTM'
    parse_action_args(args)
    args.record_for_grad = True
    args.graph_update = True
    return Trainer(args, m.make_policy(args, args.num_inputs), env)


def measure(name, flags, nenvs, updates):
    import torch
    tr = make_trainer(flags + ["--nenvs", str(nenvs), "--batch_size", "500", "--seed", "1"])
    times = {"eager": [], "graph": []}
    for u in range(updates + 1):
        for mode in ("eager", "graph"):
            tr.graph_update = mode == "graph"
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.train_batch(u)
            torch.cuda.synchronize()
            if u > 0:
                times[mode].append((time.perf_counter() - t0) * 1e3)
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    res = dict(setup=name, nenvs=nenvs, T=tr.batch_plan()[0], record_mode=tr.record_mode, grad_impl=tr.grad_impl,
               eager_ms=med["eager"], graph_ms=med["graph"], speedup=med["eager"] / med["graph"],
               eager_all_ms=times["eager"], graph_all_ms=times["graph"], captures=tr.update_captures)
    del tr
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=3)
    ap.add_argument("--only", default="")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_update.py needs a CUDA device")
    only = set(a.only.split(",")) if a.only else None
    lines = [dict(start=card())]
    print(json.dumps(lines[-1]), flush=True)
    for name, flags, n in SETUPS:
        if only and name not in only and "%s@%d" % (name, n) not in only:
            continue
        lines.append(measure(name, flags, n, a.updates))
        print(json.dumps(lines[-1]), flush=True)
    lines.append(dict(end=card()))
    print(json.dumps(lines[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
