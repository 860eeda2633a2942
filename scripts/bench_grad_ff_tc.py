"""The non-recurrent gradient kernels on the tensor cores (grad_impl 'kernels_ff_tc') against the fp32 SIMT kernels
(grad_impl 'kernels_ff'), alternated in one process over the runs of scripts/bench_grad_ff.py: models.MLP, the
non-recurrent IC3Net and the non-recurrent CommNet with 2 passes at predator-prey hard with 8192 env slots, and the
non-recurrent IC3Net at traffic-junction hard with 4096 slots; --batch_size 100 and 500 (traffic junction: 100).

    python scripts/bench_grad_ff_tc.py [--updates 2] [--rounds 1] [--batch_sizes 100,500] [--only RUN] [--out FILE]

Per measurement: train_batch and compute_grad ms per update (CUDA events), peak allocated memory, and the device time
of the backward's stages in one more compute_grad under torch.profiler (kernel records, summed over every launch):
dgrad (ff_pass_kernel | fgt_dgrad_kernel), weight gradient (ff_wgrad_kernel<false> | fgt_wgrad_kernel<false, ..>),
encoder (ff_dpre_kernel + ff_wgrad_kernel<true> | fgt_wgrad_kernel<true, ..>), and the rest (records, forward re-run,
heads, finish: the same kernels for both).  The card, its power limit and SM clock are printed first and last."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_grad_ff import RUNS, card  # noqa: E402

IMPLS = ("kernels_ff", "kernels_ff_tc")
STAGES = (("dgrad", ("ff_pass_kernel", "fgt_dgrad_kernel")),
          ("wgrad", ("ff_wgrad_kernel<false>", "fgt_wgrad_kernel<false")),
          ("encoder", ("ff_dpre_kernel", "ff_wgrad_kernel<true>", "fgt_wgrad_kernel<true")))


def build(run, grad_impl, batch_size):
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
    for k, v in dict(pol, ic3net=False, recurrent=False, rnn_type="MLP", mean_ratio=1.0, policy_impl=None, nenvs=slots,
                     record_for_grad=True, batch_size=batch_size, grad_impl=grad_impl, batch_boundary="reference",
                     value_coeff=0.01, entr=0.0, gamma=1.0, normalize_rewards=False, detach_gap=10000,
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
    assert tr.grad_ff and tr.grad_impl == grad_impl
    return tr


def stage_ms(tr, batch):
    """Device ms of the backward's stages in one compute_grad, from the profiler's kernel records."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    tr.optimizer.zero_grad(set_to_none=False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        tr.compute_grad(batch)
        torch.cuda.synchronize()
    out = dict.fromkeys([s for s, _ in STAGES] + ["other"], 0.0)
    launches = dict.fromkeys(out, 0)
    for ev in prof.key_averages():
        t = getattr(ev, "self_device_time_total", None)
        if t is None:
            t = ev.self_cuda_time_total
        if t <= 0:
            continue
        stage = next((s for s, keys in STAGES if any(k in ev.key for k in keys)), "other")
        out[stage] += t / 1e3
        launches[stage] += ev.count
    return out, launches


def measure(run, grad_impl, batch_size, opts):
    import torch

    from ic3net_b200.utils import merge_stat
    tr = build(run, grad_impl, batch_size)
    T, _ = tr.batch_plan()
    tr.train_batch(0)                                   # warm-up: allocations, weight packing
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms, grad = [], []
    for u in range(opts.updates):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        batch, stat = tr.run_batch(u + 1)               # = Trainer.train_batch, with an event before compute_grad
        ev[1].record()
        tr.optimizer.zero_grad(set_to_none=False)
        s = tr.compute_grad(batch)
        merge_stat(s, stat)
        tr.optimizer.step(grad_div=stat["num_steps"])
        ev[2].record()
        torch.cuda.synchronize()
        ms.append(ev[0].elapsed_time(ev[2]))
        grad.append(ev[1].elapsed_time(ev[2]))
    peak = torch.cuda.max_memory_allocated() / 1e9
    stages, launches = stage_ms(tr, batch)
    out = dict(run=run, grad_impl=grad_impl, env_slots=tr.env.env.nenvs, batch_size=batch_size, lock_steps=T,
               chunk_steps=tr.ff_chunk_steps, train_batch_ms=ms, compute_grad_ms=grad, peak_allocated_gb=peak,
               stage_ms=stages, stage_launches=launches)
    del tr
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=2, help="timed train_batch calls per measurement")
    ap.add_argument("--rounds", type=int, default=1, help="kernels_ff / kernels_ff_tc alternations per batch size")
    ap.add_argument("--batch_sizes", default="100,500", help="--batch_size values (lock-steps ~ this + max_steps)")
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
        for bs in (int(x) for x in opts.batch_sizes.split(",")[:1 if run.startswith("tj") else None]):
            for r in range(opts.rounds):
                for impl in IMPLS:
                    emit(dict(round=r, **measure(run, impl, bs, opts)))
    emit(dict(card_after=card()))
    if opts.out:
        with open(opts.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
