"""The IC baseline's policy step (models.RNN with the tanh recurrence, rnn_type 'MLP') on the fp32 SIMT kernel
(policy_impl 'simt', the default) against the tensor-core kernel (policy_impl 'tc_tanh', the recurrent form of ff_tc_kernel in csrc/ff_tc.cu), alternated in
one process: predator-prey hard (10 agents, dim 20, vision 1, 8192 env slots) and traffic-junction hard (20 agents,
4096 env slots), index observations, grad_impl 'kernels'.

    python scripts/bench_rnn_tc.py [--updates 3] [--rounds 2] [--batch_size 100] [--workloads pp_hard_ic3net,tj_hard_ic3net]
                                   [--out FILE]

Per measurement: rollout ms per lock-step and Trainer.train_batch ms per update (CUDA events), and the split of one
lock-step: the index encoder and the policy step timed alone over repeated launches on the trainer's own buffers, the
env step and everything else by difference from the rollout.  Prints one JSON line per measurement, and the card, its
power limit and SM clock first and last."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_bptt_rnn import card  # noqa: E402


def build(workload, impl, batch_size):
    import torch

    from bench import make_args
    from ic3net_b200 import data, models
    from ic3net_b200.action_utils import parse_action_args
    from ic3net_b200.trainer import Trainer
    a = make_args(workload, 0, "index")
    # IC: --recurrent without --commnet (models.RNN, rnn_type 'MLP'), no hard attention
    for k, v in dict(commnet=False, recurrent=True, rnn_type="MLP", hard_attn=False, mean_ratio=1.0, policy_impl=impl,
                     record_for_grad=True, batch_size=batch_size, grad_impl="kernels", batch_boundary="reference",
                     value_coeff=0.01, entr=0.0, gamma=1.0, normalize_rewards=False, detach_gap=10000,
                     comm_passes=1, share_weights=False).items():
        setattr(a, k, v)
    env = data.init(a.env_name, a)
    a.num_inputs = env.observation_dim
    a.num_actions = [env.num_actions]
    a.dim_actions = 1
    parse_action_args(a)
    torch.manual_seed(0)
    net = models.RNN(a, a.num_inputs)
    tr = Trainer(a, net, env)
    assert tr.grad_kernels and net.policy_impl == impl
    return tr


def step_split(tr, reps=50):
    """ms per launch of the index encoder and of the policy step alone, on the trainer's buffers after a rollout."""
    import torch

    from ic3net_b200 import _lib
    lib = _lib.load()
    b, e, net = tr._buf, tr.env.env, tr.policy_net
    cfg, w, s = tr._policy_cfg(), net.packed(), _lib.stream()
    ws, _ = net.workspace(e.nenvs)
    enc = lib.ic3_tj_encoder_index if tr.is_tj else lib.ic3_pp_encoder_index
    h = b["rec_h"][1] if "rec_h" in b else b["h"]
    h2, value, logp, action = (torch.empty_like(t) for t in (h, b["value"][0], b["logp"][0], b["action"][0]))
    io = _lib.PolicyIO(x=b["x"].data_ptr(), h=h.data_ptr(), c=None, comm_action=None, alive=b["alive"].data_ptr(),
                       fresh=b["fresh"].data_ptr(), tick=e.tick.data_ptr(), draws=None, h_out=h2.data_ptr(), c_out=None,
                       value=value.data_ptr(), logp=logp.data_ptr(), action=action.data_ptr(),
                       workspace=_lib.ptr(ws), err=b["err"].data_ptr())

    def timed(fn):
        for _ in range(5):
            fn()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(reps):
            fn()
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / reps

    t_enc = timed(lambda: _lib.check(enc(C.byref(e.cfg), C.byref(e.state), C.byref(cfg), C.byref(w), b["x"].data_ptr(), s)))
    t_pol = timed(lambda: _lib.check(lib.ic3_policy_step(C.byref(cfg), C.byref(w), C.byref(io), s)))
    return t_enc, t_pol


def measure(workload, impl, opts):
    import torch

    from ic3net_b200.utils import merge_stat
    tr = build(workload, impl, opts.batch_size)
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
    t_enc, t_pol = step_split(tr)
    per_step = min(roll) / T
    out = dict(policy="IC (models.RNN, tanh)", workload=workload, policy_impl=impl, env_slots=tr.env.env.nenvs,
               rows=tr.env.env.nenvs * tr.args.nagents, batch_size=opts.batch_size, lock_steps=T,
               record_mode=tr.record_mode, ms_per_update=ms, rollout_ms=roll,
               rollout_ms_per_lock_step=[r / T for r in roll],
               split_ms_per_lock_step=dict(index_encoder=t_enc, policy_step=t_pol,
                                           env_step_and_rest_by_difference=per_step - t_enc - t_pol))
    del tr
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=3, help="timed train_batch calls per measurement")
    ap.add_argument("--rounds", type=int, default=2, help="simt / tc_tanh alternations per workload")
    ap.add_argument("--batch_size", type=int, default=100, help="--batch_size (lock-steps ~ this + max_steps)")
    ap.add_argument("--workloads", default="pp_hard_ic3net,tj_hard_ic3net", help="bench.py workload geometries")
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
    for wl in opts.workloads.split(","):
        for r in range(opts.rounds):
            for impl in ("simt", "tc_tanh"):
                emit(dict(round=r, **measure(wl, impl, opts)))
    emit(dict(card_after=card()))
    if opts.out:
        with open(opts.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
