"""Trainer.evaluate throughput: whole episodes per second and agent-env-steps per second, at predator-prey hard IC3Net
(8192 slots) and traffic-junction hard IC3Net (4096 slots), sampled and greedy, eager and replayed as a CUDA graph
(--use_graph).  Then the success rate of sampled and greedy evaluation after a few training updates (reported, not
asserted).

    python scripts/bench_eval.py [--episodes 2] [--repeats 3] [--train 5] [--out FILE]

Each evaluate call is timed by the host clock up to its device->host read of the statistics (the call ends in a
synchronise).  The first call of each mode (and the graph capture) is warm-up and not timed.  Prints one JSON line per
measurement, and the card, its power limit and SM clock first and last."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_graph_update import IC3NET, PP, TJ, card, make_trainer  # noqa: E402

SETUPS = [("pp_hard_ic3net", PP + IC3NET, 8192), ("tj_hard_ic3net", TJ + IC3NET, 4096)]


def measure(name, flags, nenvs, episodes, repeats, train):
    import torch
    tr = make_trainer(flags + ["--nenvs", str(nenvs), "--batch_size", "500", "--seed", "1"])
    tr.graph_update = False
    out = []
    for graph in (False, True):
        tr.use_graph = graph
        for greedy in (False, True):
            tr.evaluate(episodes, greedy)                    # warm-up (and capture)
            times, st = [], None
            for _ in range(repeats):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                st = tr.evaluate(episodes, greedy)
                times.append(time.perf_counter() - t0)
            s = sorted(times)[len(times) // 2]
            out.append(dict(setup=name, nenvs=nenvs, episodes_per_slot=episodes, graph=graph, greedy=greedy,
                            seconds=s, episodes_per_s=st["num_episodes"] / s,
                            agent_env_steps_per_s=st["num_steps"] * tr.args.nagents / s,
                            success_rate=st.get("success", 0) / st["num_episodes"], all_seconds=times))
    tr.use_graph = False
    for u in range(train):
        tr.train_batch(u)
    for greedy in (False, True):
        st = tr.evaluate(episodes, greedy)
        out.append(dict(setup=name, after_updates=train, greedy=greedy,
                        success_rate=st.get("success", 0) / st["num_episodes"],
                        steps_per_episode=st["num_steps"] / st["num_episodes"]))
    del tr
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--episodes", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--train", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py needs a CUDA device")
    lines = [dict(start=card())]
    print(json.dumps(lines[-1]), flush=True)
    for name, flags, n in SETUPS:
        for r in measure(name, flags, n, a.episodes, a.repeats, a.train):
            lines.append(r)
            print(json.dumps(r), flush=True)
    lines.append(dict(end=card()))
    print(json.dumps(lines[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
