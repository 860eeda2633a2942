"""What recording messages costs: Trainer.evaluate_trace without and with messages=True (K = 8 slots, with and without
the comm map, which turns the message map on), eager and replayed as a CUDA graph (--use_graph), at predator-prey hard
IC3Net (8192 slots) and traffic-junction hard IC3Net (4096 slots).

    python scripts/bench_eval_messages.py [--episodes 1] [--repeats 3] [--out FILE]

Every call is timed by the host clock up to its device->host reads (the call ends in a synchronise).  For each
configuration, the recording without and with messages run once untimed (warm-up and graph capture), then alternate
for the timed rounds in one process; the medians are reported with the difference per lock-step.  Prints one JSON line
per measurement, and the card, its power limit and SM clock first and last."""
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


def measure(name, flags, nenvs, episodes, repeats):
    import torch
    tr = make_trainer(flags + ["--nenvs", str(nenvs), "--batch_size", "500", "--seed", "1"])
    tr.graph_update = False
    out = []
    T = episodes * tr.args.max_steps
    for graph in (False, True):
        tr.use_graph = graph
        for cmap in (False, True):
            # the recorder (and its graph) is rebuilt when the message switch changes, as it is for any new
            # configuration; alternating the two therefore times each with its own allocation and capture, so each
            # mode gets a trainer of its own
            pair = (tr, make_trainer(flags + ["--nenvs", str(nenvs), "--batch_size", "500", "--seed", "1"]))
            pair[1].graph_update = False
            pair[1].use_graph = graph
            modes = (lambda: pair[0].evaluate_trace(episodes, slots=8, comm_map=cmap),
                     lambda: pair[1].evaluate_trace(episodes, slots=8, comm_map=cmap, messages=True))
            times = ([], [])
            for f in modes:
                f()                                      # warm-up (and capture)
            for _ in range(repeats):
                for f, ts in zip(modes, times):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    f()
                    ts.append(time.perf_counter() - t0)
            base, s = (sorted(ts)[repeats // 2] for ts in times)
            out.append(dict(setup=name, nenvs=nenvs, episodes_per_slot=episodes, graph=graph, slots=8, comm_map=cmap,
                            trace_seconds=base, messages_seconds=s, ms_per_lockstep=1e3 * s / T,
                            overhead_us_per_lockstep=1e6 * (s - base) / T, trace_all=times[0],
                            messages_all=times[1]))
            del pair
            torch.cuda.empty_cache()
    del tr
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--episodes", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_messages.py needs a CUDA device")
    lines = [dict(start=card())]
    print(json.dumps(lines[-1]), flush=True)
    for name, flags, n in SETUPS:
        for r in measure(name, flags, n, a.episodes, a.repeats):
            lines.append(r)
            print(json.dumps(r), flush=True)
    lines.append(dict(end=card()))
    print(json.dumps(lines[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
