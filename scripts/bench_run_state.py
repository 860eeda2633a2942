"""Size and write time of the run-state sidecar of --resumable (main.py save_checkpoint with ``run``), at
predator-prey hard IC3Net (8192 slots) and traffic-junction hard IC3Net (4096 slots), with the evaluation env built.

    python scripts/bench_run_state.py [--repeats 5] [--out FILE]

Times, by the host clock, Trainer.run_state() (device->host copies of the env states) and the whole save of the
checkpoint and its sidecar into a temporary directory, median of the repeats after one warm-up.  The bytes of the env
state are computed from the snapshot shapes.  Prints one JSON line per setup, and the card, its power limit and SM
clock first and last."""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_graph_update import IC3NET, PP, TJ, card, make_trainer  # noqa: E402

SETUPS = [("pp_hard_ic3net", PP + IC3NET, 8192), ("tj_hard_ic3net", TJ + IC3NET, 4096)]


def state_bytes(e):
    return sum(getattr(e, k).numel() * getattr(e, k).element_size() for k in e._STATE)


def measure(name, flags, nenvs, repeats):
    import torch
    from ic3net_b200 import main as m
    tr = make_trainer(flags + ["--nenvs", str(nenvs), "--batch_size", "500", "--seed", "1"])
    tr.evaluate(1)                                           # builds the evaluation env, whose state is saved too
    log = m.make_log()
    rs, save = [], []
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "ck.pt")
        for i in range(repeats + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            state = tr.run_state()
            t1 = time.perf_counter()
            m.save_checkpoint(path, tr.policy_net, log, tr, None, dict(ep=1, update=0, stat=None, state=state))
            t2 = time.perf_counter()
            if i:
                rs.append(t1 - t0)
                save.append(t2 - t1)
        sizes = dict(checkpoint_bytes=os.path.getsize(path), sidecar_bytes=os.path.getsize(path + ".run"))
    med = lambda v: sorted(v)[len(v) // 2]
    out = dict(setup=name, nenvs=nenvs, train_env_state_bytes=state_bytes(tr.env.env),
               eval_env_state_bytes=state_bytes(tr._eval["env"]), run_state_seconds=med(rs),
               save_pair_seconds=med(save), all_run_state_seconds=rs, all_save_pair_seconds=save, **sizes)
    del tr
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_run_state.py needs a CUDA device")
    lines = [dict(start=card())]
    print(json.dumps(lines[-1]), flush=True)
    for name, flags, n in SETUPS:
        lines.append(measure(name, flags, n, a.repeats))
        print(json.dumps(lines[-1]), flush=True)
    lines.append(dict(end=card()))
    print(json.dumps(lines[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
