"""The BPTT kernels (csrc/bptt_tc.cu) on the tanh RNN without communication: models.RNN with rnn_type 'MLP', the IC and
IRIC baselines (IRIC = IC with mean_ratio 0), which run on the SIMT policy kernel.

Covered:
  - the gradient against a float64 backward over the kernel trainer's own records (h alone): every step re-run in
    float64 from rec_h[t], the heads' backward started from the recorded log-probs and values as the kernels' is, the
    recursion carried step by step; on ragged tiles, at row counts around the thresholds of the tanh, dgrad and
    weight-gradient kernels (from the card's SM count), and at the full batch sizes;
  - a cross-check against the torch-autograd windowed recompute of the same rollout;
  - bit-identical gradients run to run, between the two-stream and the one-stream schedule, between full and windowed
    records;
  - the refusals (tanh cells with communication, models.MLP, the non-recurrent CommNet, a 7x7 window, an observation
    pattern wider than 512 columns) and train_batch end to end.

Bar against float64: that of tests/test_gpu_bptt_kernels.py: per tensor 1e-4 of its largest entry (affine1.weight also
per input column), the action heads also 2^-20 of their sum of |terms|; loss sums rtol 2e-4.  Against autograd: the bar
of tests/test_gpu_bptt_passes.py."""
import ctypes as C
import math

import pytest
import torch

from bptt_ref import LOSS_KEYS
from gpu_harness import (PP, TJ, events, grads_of, kernels_vs_autograd, one_stream_schedule, rnn_full_size,
                         rnn_gradient_arrays, rnn_pinned_oracle, rnn_records_reference as records_reference,
                         rnn_run_to_run, rnn_trainer as make_trainer, rnn_windows, trainer_within_bar)
from helpers import golden_names, load_golden

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------- the reference

@pytest.mark.parametrize("B", [5, 13])
@pytest.mark.parametrize("name", golden_names("gradrnn_"))
def test_kernels_match_reference_pinned_oracle(name, B):
    rnn_pinned_oracle(name, B, None)


@pytest.mark.parametrize("name", golden_names("gradrnn_"))
def test_kernels_match_reference_gradient_arrays(name):
    rnn_gradient_arrays(name, None)


# ---------------------------------------------------------------------------------------------------- vs float64

CASES = {
    "pp_ic_detach": (PP, dict(detach_gap=4, max_steps=12, batch_size=30)),
    "tj_iric": (TJ, dict(mean_ratio=0.0)),
    "pp_ic_enemy_entr": ("grad_pp_enemy_ic3net_h128", dict(entr=0.01, normalize_rewards=True)),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("B", [5, 13])
def test_gradient_matches_float64_records(case, B):
    """B * N never a multiple of 128: a ragged last tile."""
    name, over = CASES[case]
    tr = make_trainer(name, B, **over)
    assert tr.grad_kernels and tr.grad_impl == "kernels" and tr.record_mode == "full"
    tr.run_batch(0)
    got, gloss = grads_of(tr)
    ref, rloss = records_reference(tr)
    ev = events(tr)
    if case == "pp_ic_detach":                       # 12-step episodes inside a 30-step quota: restarts and cuts
        assert ev["fresh"] > 0 and ev["cut"] > 0, ev
    assert int(tr._buf["err"].item()) == 0
    trainer_within_bar(tr, got, gloss, ref, rloss, "%s B=%d %s" % (case, B, ev))


@pytest.mark.parametrize("name,B", [(PP, 8192), (TJ, 4096)])
def test_full_size_gradient_matches_float64(name, B):
    rnn_full_size(name, B, None)


def _split(np_cols, sms):
    """(j0, j1) of the weight-gradient kernel for one 128-column gate block with the h block as slice 0 (plan_layout)."""
    per_mb = sms // 2
    c0 = 3.0 * (128 + 86) / 3.0
    c1 = 2.0 * (128 + 0.5 * (np_cols - 256) + 22 if np_cols > 256 else 0.5 * np_cols + 22)
    j0 = min(max(int(per_mb * c0 / (c0 + c1) + 0.5), 1), per_mb - 1)
    return j0, per_mb - j0


@pytest.mark.parametrize("case", ["R<16", "R=128k+2", "dgrad-2-tiles", "wgrad-uneven"])
def test_row_counts_around_thresholds(case):
    """Predator-prey hard geometry (10 agents): fewer rows than one block of the tanh kernel, two rows in the last tile,
    dgrad CTAs with two tiles (> SMs tiles), and a tile count neither weight-gradient slice's role count divides."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    N = load_golden(PP)[0]["args"]["nagents"]
    probe = make_trainer(PP, 1)
    e = probe.env.env
    W = 2 * e.vision + 1
    np_cols = (e.obs_positions + 2 * W * W + 1 + 15) // 16 * 16
    j0, j1 = _split(np_cols, sms)
    if case == "R<16":
        B = 1
    elif case == "R=128k+2":
        B = next(b for b in range(13, 10000) if (b * N) % 128 == 2)
    elif case == "dgrad-2-tiles":
        B = next(b for b in range(sms * 128 // N, 100000) if -(-b * N // 128) > sms and (b * N) % 128)
    else:
        B = next(b for b in range(j0 * 128 // N + 1, 100000)
                 if -(-b * N // 128) % j0 and -(-b * N // 128) % j1 and -(-b * N // 128) > j0 + j1)
    tr = make_trainer(PP, B, seed=77, id0=3, batch_size=14, max_steps=10, detach_gap=3)
    R = B * N
    nt = -(-R // 128)
    tr.run_batch(0)
    got, gloss = grads_of(tr)
    ref, rloss = records_reference(tr)
    trainer_within_bar(tr, got, gloss, ref, rloss, "%s: B=%d R=%d tiles=%d j0=%d j1=%d SMs=%d" % (case, B, R, nt, j0, j1,
                                                                                               sms))


# ---------------------------------------------------------------------------------------------------- vs autograd

@pytest.mark.parametrize("name,over", [(PP, dict(detach_gap=3, max_steps=8)), (TJ, dict(mean_ratio=0.0))])
def test_gradient_matches_autograd(name, over):
    tk = make_trainer(name, 64, **over)
    ta = make_trainer(name, 64, grad_impl="autograd", **over)
    kernels_vs_autograd(tk, ta, "%s %s" % (name, over))


# ---------------------------------------------------------------------------------------------------- determinism

def test_one_stream_schedule_is_bit_identical(tmp_path):
    one_stream_schedule(tmp_path, "gpu_harness", "schedule_rnn", more_than=3)


def test_repeated_compute_grad_is_bit_identical():
    rnn_run_to_run(None)


@pytest.mark.parametrize("name,window", [(PP, 4), (TJ, 1)])
def test_windowed_records_are_bit_identical(name, window):
    rnn_windows(name, window, None)


def test_records_hold_h_alone():
    """At predator-prey hard, 8192 slots, batch 500 the full records are (T + 1) B N H float32: 24.3 GB, half the LSTM's."""
    tr = make_trainer(PP, 8192, batch_size=500, max_steps=80, mode="mixed")
    T = tr.batch_plan()[0]
    assert T == 579
    nbytes = tr._record_bytes(T)["full"]
    assert nbytes == (T + 1) * 8192 * 10 * 128 * 4
    assert abs(nbytes / 1e9 - 24.3) < 0.05, nbytes


# ---------------------------------------------------------------------------------------------------- refusals

@pytest.mark.parametrize("model,over", [("mlp", {}), ("commnet", dict(commnet=True, recurrent=False, comm_passes=2)),
                                        ("rnn", dict(vision=3)), ("rnn", dict(dim=22, vision=2))])
def test_out_of_scope_configurations_fall_back(model, over):
    """models.MLP, the non-recurrent CommNet (tanh cells with x_tanh / h_from_x), a 7x7 window and an observation
    pattern of more than 512 columns: 'kernels' raises, 'auto' takes autograd."""
    kw = dict(over, model=model)
    if model == "commnet":
        kw["policy_impl"] = "simt"
    with pytest.raises(NotImplementedError):
        make_trainer(PP, 8, **kw)
    tr = make_trainer(PP, 8, grad_impl="auto", **kw)
    assert not tr.grad_kernels and tr.grad_impl == "autograd" and tr.record_mode is None


def test_tanh_cell_with_communication_gets_no_workspace():
    """The library sizes the tanh cell only without communication: comm_mask_zero = 0, hard attention or two passes
    give 0 bytes; the in-scope configuration is sized."""
    from ic3net_b200 import _lib
    lib = _lib.load()
    hd = (C.c_int32 * _lib.MAX_HEADS)(5, 0, 0, 0)
    pol = dict(B=4, N=3, H=128, O=9 * 13, nheads=1, head_dim=hd, hard_attn=0, comm_avg=1, comm_mask_zero=1, env_id0=0, seed=1,
               obs_off=0, obs_vocab=13, obs_ncount=2, cell=_lib.CELL_TANH, passes=1, x_tanh=0, h_from_x=0)
    env = _lib.PPCfg(B=4, N=3, dim=3, vision=1, mode=0, naction=5, env_id0=0, enemy_comm=0, seed=1)

    def nbytes(**kw):
        cfg = _lib.PolicyCfg(**dict(pol, **kw))
        plan = _lib.BpttPlan(cfg=C.pointer(cfg), w=None, pp_env=C.pointer(env), tj_env=None, x_table=None,
                             value_coeff=0.01, entr=0.0, workspace=None)
        return int(lib.ic3_bptt_workspace_bytes(C.byref(plan)))

    for bad in (dict(comm_mask_zero=0), dict(hard_attn=1), dict(passes=2), dict(H=64)):
        assert nbytes(**bad) == 0, bad
    assert nbytes() > 0


# ---------------------------------------------------------------------------------------------------- end to end

@pytest.mark.parametrize("name,mean_ratio", [(PP, 1.0), (PP, 0.0), (TJ, 1.0), (TJ, 0.0)])
def test_train_batch_ic_iric(name, mean_ratio):
    """IC (mean_ratio 1) and IRIC (mean_ratio 0) under grad_impl 'auto': the kernels, finite losses, parameters move."""
    tr = make_trainer(name, 64, grad_impl="auto", mean_ratio=mean_ratio, detach_gap=5)
    assert tr.grad_impl == "kernels" and tr.grad_kernels
    before = tr.optimizer.flat_params.clone()
    for ep in range(2):
        stat = tr.train_batch(ep)
        assert all(math.isfinite(stat[k]) for k in LOSS_KEYS), stat
    assert not torch.equal(before, tr.optimizer.flat_params)
    assert int(tr._buf["err"].item()) == 0
