"""The non-recurrent tanh policies' step (models.MLP, CommNet / IC3Net without --recurrent) on the fp32 SIMT kernel
(policy_impl 'simt', the default) against the tensor-core kernel (policy_impl 'tc_ff', csrc/ff_tc.cu), alternated in one
process: predator-prey hard (10 agents, dim 20, vision 1, 8192 env slots) with MLP, IC3Net and CommNet with 2 passes,
and traffic-junction hard (20 agents, 4096 env slots) with IC3Net; index observations, grad_impl 'kernels_ff'.

    python scripts/bench_ff_tc.py [--updates 3] [--rounds 2] [--batch_size 100] [--cases pp_mlp,pp_ic3net,pp_commnet2,tj_ic3net]
                                  [--out FILE]

Per measurement (CUDA events): the policy step alone over 50 launches on the trainer's own buffers, the rollout per
lock-step, Trainer.train_batch ms per update, the gradient (compute_grad) ms, and the forward re-run of the kernels_ff
backward: ic3_policy_ff_states over one lock-step's slots timed alone, times the lock-steps of the batch (the re-run is
one launch sequence per chunk over K lock-steps' rows; its cost is linear in the rows), as a share of compute_grad.
Prints one JSON line per measurement, and the card, its power limit and SM clock first and last."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_bptt_rnn import card  # noqa: E402

CASES = {
    "pp_mlp": ("pp_hard_ic3net", "mlp", 1),
    "pp_ic3net": ("pp_hard_ic3net", "ic3net", 1),
    "pp_commnet2": ("pp_hard_ic3net", "commnet", 2),
    "tj_ic3net": ("tj_hard_ic3net", "ic3net", 1),
}


def build(case, impl, batch_size):
    import torch

    from bench import make_args
    from ic3net_b200 import data, models
    from ic3net_b200.action_utils import parse_action_args
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    workload, family, passes = CASES[case]
    a = make_args(workload, 0, "index")
    for k, v in dict(commnet=family != "mlp", recurrent=False, rnn_type="MLP", hard_attn=family == "ic3net",
                     mean_ratio=1.0, policy_impl=impl, record_for_grad=True, batch_size=batch_size, grad_impl="kernels_ff",
                     batch_boundary="reference", value_coeff=0.01, entr=0.0, gamma=1.0, normalize_rewards=False,
                     detach_gap=10000, comm_passes=passes, share_weights=False).items():
        setattr(a, k, v)
    env = data.init(a.env_name, a)
    a.num_inputs = env.observation_dim
    a.num_actions = [env.num_actions]
    a.dim_actions = 1
    parse_action_args(a)
    torch.manual_seed(0)
    net = (models.MLP if family == "mlp" else CommNetMLP)(a, a.num_inputs)
    tr = Trainer(a, net, env)
    assert tr.grad_ff and net.policy_impl == impl
    return tr


def timed(fn, reps=50):
    import torch
    for _ in range(5):
        fn()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def step_split(tr):
    """ms per launch of the index encoder, the policy step and the pass-state re-run, on the trainer's buffers."""
    import torch

    from ic3net_b200 import _lib
    lib = _lib.load()
    b, e, net = tr._buf, tr.env.env, tr.policy_net
    cfg, w, s = tr._policy_cfg(), net.packed(), _lib.stream()
    ws, _ = net.workspace(e.nenvs)
    enc = lib.ic3_tj_encoder_index if tr.is_tj else lib.ic3_pp_encoder_index
    R, H, P = e.nenvs * tr.args.nagents, tr.args.hid_size, max(1, int(cfg.passes))
    h2 = torch.empty(R, H, device="cuda")
    value, logp, action = (torch.empty_like(t) for t in (b["value"][0], b["logp"][0], b["action"][0]))
    comm = b["comm"].data_ptr() if tr.hard else None
    io = _lib.PolicyIO(x=b["x"].data_ptr(), h=None, c=None, comm_action=comm, alive=b["alive"].data_ptr(),
                       fresh=b["fresh"].data_ptr(), tick=e.tick.data_ptr(), draws=None, h_out=h2.data_ptr(), c_out=None,
                       value=value.data_ptr(), logp=logp.data_ptr(), action=action.data_ptr(),
                       workspace=_lib.ptr(ws), err=b["err"].data_ptr())
    st_h = torch.empty(P + 1, R, H, device="cuda")
    st_s = torch.empty(P, R, H, device="cuda") if not cfg.comm_mask_zero else None
    sio = _lib.PolicyIO(x=b["x"].data_ptr(), comm_action=comm, alive=b["alive"].data_ptr(), fresh=b["fresh"].data_ptr())
    t_enc = timed(lambda: _lib.check(enc(C.byref(e.cfg), C.byref(e.state), C.byref(cfg), C.byref(w), b["x"].data_ptr(), s)))
    t_pol = timed(lambda: _lib.check(lib.ic3_policy_step(C.byref(cfg), C.byref(w), C.byref(io), s)))
    t_st = timed(lambda: _lib.check(lib.ic3_policy_ff_states(C.byref(cfg), C.byref(w), C.byref(sio), st_h.data_ptr(),
                                                             _lib.ptr(st_s), s)))
    return t_enc, t_pol, t_st


def measure(case, impl, opts):
    import torch

    from ic3net_b200.utils import merge_stat
    tr = build(case, impl, opts.batch_size)
    T, _ = tr.batch_plan()
    tr.train_batch(0)                                   # warm-up: allocations, weight packing
    torch.cuda.synchronize()
    ms, roll, grad = [], [], []
    for u in range(opts.updates):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        batch, stat = tr.run_batch(u + 1)               # = Trainer.train_batch, with events after rollout and gradient
        ev[1].record()
        tr.optimizer.zero_grad(set_to_none=False)
        s = tr.compute_grad(batch)
        ev[2].record()
        merge_stat(s, stat)
        tr.optimizer.step(grad_div=stat["num_steps"])
        ev[3].record()
        torch.cuda.synchronize()
        assert int(tr._buf["err"].item()) == 0
        ms.append(ev[0].elapsed_time(ev[3]))
        roll.append(ev[0].elapsed_time(ev[1]))
        grad.append(ev[1].elapsed_time(ev[2]))
    t_enc, t_pol, t_st = step_split(tr)
    per_step = min(roll) / T
    out = dict(case=case, workload=CASES[case][0], family=CASES[case][1], comm_passes=CASES[case][2], policy_impl=impl,
               env_slots=tr.env.env.nenvs, rows=tr.env.env.nenvs * tr.args.nagents, batch_size=opts.batch_size,
               lock_steps=T, ff_chunk_steps=tr.ff_chunk_steps, ms_per_update=ms, rollout_ms=roll,
               rollout_ms_per_lock_step=[r / T for r in roll], compute_grad_ms=grad,
               split_ms_per_lock_step=dict(index_encoder=t_enc, policy_step=t_pol,
                                           env_step_and_rest_by_difference=per_step - t_enc - t_pol),
               rerun_ms_per_lock_step=t_st, rerun_share_of_compute_grad=t_st * T / min(grad))
    del tr
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--updates", type=int, default=3, help="timed train_batch calls per measurement")
    ap.add_argument("--rounds", type=int, default=2, help="simt / tc_ff alternations per case")
    ap.add_argument("--batch_size", type=int, default=100, help="--batch_size (lock-steps ~ this + max_steps)")
    ap.add_argument("--cases", default=",".join(CASES), help="subset of " + ", ".join(CASES))
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
    for case in opts.cases.split(","):
        for r in range(opts.rounds):
            for impl in ("simt", "tc_ff"):
                emit(dict(round=r, **measure(case, impl, opts)))
    emit(dict(card_after=card()))
    if opts.out:
        with open(opts.out, "a") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
