"""GPU tests of the BPTT kernels with windowed (h, c) records (``Trainer.record_mode == 'window'``): the rollout keeps
(h, c) only at the starts of ``grad_window``-step windows, and the backward re-runs the tensor-core policy step over
one window at a time from its checkpoint (``Trainer._recompute_window``) just ahead of the BPTT kernels.

Windows are forced at small sizes with ``Trainer.RECORD_BYTES_LIMIT = 0`` (full records never fit).  Covered: the
gradient and loss sums bit-identical to full records (full batch sizes, ragged / one-step / single windows, episode
starts and detach_gap cuts on window starts, enemy_comm, hard attention off, dense and index observations, eager and
CUDA-graph rollouts, the one-stream schedule), every recomputed window equal to the full record bit for bit, the
reference fixtures against the float64 oracle, a batch whose full records do not fit on the card, and the selection."""
import numpy as np
import pytest
import torch

from bptt_ref import LOSS_KEYS, max_rel_err, oracle_grad_sum, returns_and_advantages, trainer_reference
from gpu_harness import (LOSS_ATOL, LOSS_RTOL, SUM_FLOOR, TOL, flat_grad, lstm_fixture_weights,
                         lstm_trainer as make_trainer, one_stream_schedule, window_vs_full)
from helpers import golden_names, load_golden
from oracle import policy as opolicy

pytestmark = pytest.mark.gpu


def boundary_events(tr, W):
    """(episode starts, detach_gap cuts) that fall on window starts: fresh slots at t = kW, and cuts after step
    kW - 1 (the state entering window k detached)."""
    b, args = tr._buf, tr.args
    T = b["T"]
    fresh = int(b["s_fresh"][W::W].sum())
    cut = int((((b["s_tep"][W - 1:T - 1:W] + 1) % args.detach_gap) == 0).sum()) if args.detach_gap <= args.max_steps \
        else 0
    return fresh, cut


# ---------------------------------------------------------------------------------------------------- bit equality

@pytest.mark.parametrize("name,B,W,over", [
    # T = 30: seven windows of 4, then 2; episodes of 20 steps start on a window start, detach_gap 8 cuts after step 7
    ("grad_pp_hard_ic3net_h128", 8192, 4, dict(batch_size=11)),
    # T = 50: ten windows of 5; the second episode starts at step 25, detach_gap 10 cuts after steps 9, 19, 34, 44
    ("grad_tj_hard_ic3net_h128", 4096, 5, {}),
])
def test_full_size_windows_are_bit_identical(name, B, W, over):
    _, tf = window_vs_full(name, B, W, **over)
    fresh, cut = boundary_events(tf, W)
    print(name, "T", tf._buf["T"], "episode starts / cuts on window starts:", fresh, cut)
    assert fresh > 0 and cut > 0
    assert tf.is_tj or int((tf._buf["valid"] == 0).sum()) > 0           # halted slots (reference batch boundary)


SMALL = {
    "one-step windows": ("grad_pp_hard_ic3net_h128", 400, 1, {}),
    "one window": ("grad_pp_hard_ic3net_h128", 400, 64, {}),
    "ragged": ("grad_pp_hard_ic3net_h128", 400, 5, {}),
    "ragged, graph": ("grad_pp_hard_ic3net_h128", 400, 5, dict(use_graph=True)),
    "hard attention off": ("grad_pp_v1_commnet_entr_h128", 400, 4, {}),
    "enemy_comm": ("grad_pp_enemy_ic3net_h128", 400, 4, {}),
    "dense, side-stream writer": ("grad_pp_hard_ic3net_h128", 400, 5, dict(obs_mode="dense")),
    "dense, gather + encoder, graph": ("grad_pp_enemy_ic3net_h128", 64, 3, dict(obs_mode="dense", use_graph=True)),
    "tj dense, graph": ("grad_tj_medium_v1_ic_h128", 400, 6, dict(obs_mode="dense", use_graph=True)),
}


@pytest.mark.parametrize("case", list(SMALL))
def test_windows_are_bit_identical(case):
    name, B, W, over = SMALL[case]
    _, tf = window_vs_full(name, B, W, **over)
    if case.startswith("dense"):
        assert "obs" in tf._buf and tf._overlap_obs() == ("side-stream" in case)
    if case == "one window":
        assert tf._buf["T"] <= W


def test_one_stream_schedule(tmp_path):
    """IC3_BPTT_OVERLAP=0 (read once per process: a child) runs the look-ahead kernels on the caller's stream, behind
    the recompute of every window: still bit-identical to full records, and to the two-stream schedule."""
    files = one_stream_schedule(tmp_path, "gpu_harness", "schedule_windows", more_than=3)
    assert len(files) == 4


# ---------------------------------------------------------------------------------------------------- reference

H128 = [n for n in golden_names("grad_") if load_golden(n)[0]["args"]["hid_size"] == 128]


@pytest.mark.parametrize("name", H128)
def test_windows_match_oracle(name):
    """Every hid_size-128 gradient fixture in window mode (4-step windows) against the float64 oracle's sum over the
    slots, at the bar of the full-record kernels (test_gpu_grad.py)."""
    B, seed, id0 = 5, 808, 30
    tr = make_trainer(name, B, seed, id0, windows=True, grad_window=4)
    meta, z = load_golden(name)
    sd = lstm_fixture_weights(meta, tr.args)
    batch, stat = tr.run_batch(0)
    assert tr.record_mode == "window"
    T, quota = tr.batch_plan()
    tr.optimizer.zero_grad(set_to_none=False)
    s = tr.compute_grad(batch)
    want, wstat, nsteps = oracle_grad_sum(tr.args, z, opolicy.params_to_f64(sd), batch.action.cpu().numpy(),
                                          batch.valid.cpu().numpy(), seed, id0, quota, T)
    assert stat["num_steps"] == nsteps
    for q in LOSS_KEYS:
        assert np.isclose(s[q], wstat[q], rtol=LOSS_RTOL, atol=LOSS_ATOL), (q, s[q], wstat[q])
    worst = 0.0
    for key, prm in tr.policy_net.named_parameters():
        if want[key] is None or not np.any(want[key]):
            assert prm.grad is None or float(prm.grad.abs().max()) == 0.0, key
            continue
        err = max_rel_err(prm.grad.detach().cpu().numpy(), want[key])
        worst = max(worst, err)
        assert err < TOL, (name, key, err)
    print(name, "window mode: worst relative gradient error %.2e" % worst)


# ---------------------------------------------------------------------------------------------------- the lifted limit

class _SlotRecords(object):
    """rec_h / rec_c stand-in for tests/bptt_ref.trainer_reference restricted to single env slots: [t, rows of slot k]
    -> the (h, c) of slot k entering step t, gathered from the window recompute."""

    def __init__(self, per_slot, N):
        self.per_slot, self.N = per_slot, N

    def __getitem__(self, idx):
        t, rows = idx
        return self.per_slot[rows.start // self.N][t]


class _WithRecords(object):
    """The trainer as trainer_reference sees it, with per-slot records in place of the full ones."""

    def __init__(self, tr, rec_h, rec_c):
        self._tr = tr
        self._buf = dict(tr._buf, rec_h=rec_h, rec_c=rec_c)

    def __getattr__(self, k):
        return getattr(self._tr, k)


def slot_records(tr, slots):
    """{slot: [T+1, N, H]} of h and of c entering each step (entry 0: checkpoint 0), from the window recompute."""
    b, N, W = tr._buf, tr.args.nagents, tr.grad_window
    T = b["T"]
    hs = {k: [b["ck_h"][0][k * N:(k + 1) * N].clone()] for k in slots}
    cs = {k: [b["ck_c"][0][k * N:(k + 1) * N].clone()] for k in slots}
    for w in range((T + W - 1) // W):
        wh, wc = tr._recompute_window(w)
        for k in slots:
            hs[k].extend(wh[:, k * N:(k + 1) * N].clone().unbind(0))
            cs[k].extend(wc[:, k * N:(k + 1) * N].clone().unbind(0))
    return ({k: torch.stack(v) for k, v in hs.items()}, {k: torch.stack(v) for k, v in cs.items()})


def slot_heads_abs_sums(tr, rec_h, slots):
    """tests/bptt_ref.heads_abs_sums over the rows of ``slots`` (h' from the per-slot records)."""
    b, args = tr._buf, tr.args
    T, N = b["T"], args.nagents
    f64 = torch.float64
    _, adv = returns_and_advantages(tr)
    out = {}
    for k in slots:
        for t in range(T):
            a = (-adv[t, k].reshape(N, 1) * b["ralive"][t, k].reshape(N, 1)).to(f64)
            vrow = b["valid"][t, k].to(f64).expand(N, 1)
            h2 = rec_h.per_slot[k][t + 1].to(f64).abs()
            lp_all = b["logp"][t, k].reshape(N, -1).to(f64)
            act = b["action"][t, k].long().reshape(N, -1)
            off = 0
            for m, na in enumerate(args.naction_heads):
                lp = lp_all[:, off:off + na]
                p = lp.exp()
                g = a * (torch.zeros_like(p).scatter_(1, act[:, m:m + 1], 1.0) - p)
                if args.entr > 0:
                    g = g + args.entr * p * (lp - (p * lp).sum(1, keepdim=True)) * vrow
                g = g.abs()
                for key, v in (("heads.%d.bias" % m, g.sum(0)), ("heads.%d.weight" % m, g.t() @ h2)):
                    out[key] = out[key] + v if key in out else v
                off += na
    return out


PEAK_BOUND = 20e9           # bytes (16.1 GB measured on an H100 80GB HBM3); full records alone would take 90.6 GB


def test_batch_beyond_full_records_trains():
    """Predator-prey hard, 8192 env slots, --batch_size 1000 (T = 1079 lock-steps): full records would take 90.6 GB,
    more than the card holds, so the default selection picks windows.  A real train_batch completes with finite
    gradients and statistics under PEAK_BOUND; then, on the next batch, the kernels' gradient of 5 sampled slots and
    the last slot (the other slots' learning signal masked out) matches the float64 reference over those slots."""
    B = 8192
    tr = make_trainer("grad_pp_hard_ic3net_h128", B, seed=5, id0=0, batch_size=1000, max_steps=80)
    T, _ = tr.batch_plan()
    assert T == 1079 and tr._record_bytes(T)["full"] > torch.cuda.get_device_properties(0).total_memory
    assert tr.record_mode == "window"
    torch.cuda.reset_peak_memory_stats()
    stat = tr.train_batch(0)
    peak = torch.cuda.max_memory_allocated()
    assert tr.record_mode == "window"
    print("train_batch at T = %d: peak %.2f GB, %d steps" % (T, peak / 1e9, stat["num_steps"]))
    assert peak < PEAK_BOUND
    assert stat["num_steps"] >= B * 1000
    assert all(np.isfinite(stat[k]) for k in LOSS_KEYS)
    assert bool(torch.isfinite(tr.optimizer.flat_grads).all()) and bool(torch.isfinite(tr.optimizer.flat_params).all())

    tr.run_batch(1)
    slots = sorted(set(np.random.RandomState(0).choice(B - 1, 5, replace=False).tolist()) | {B - 1})
    b = tr._buf
    keep = torch.zeros(B, dtype=torch.bool, device="cuda")
    keep[slots] = True
    b["valid"].mul_(keep.to(torch.uint8))                       # no loss, no gradient from the other slots
    b["ralive"].mul_(keep.view(1, B, 1).to(torch.uint8))
    tr.optimizer.zero_grad(set_to_none=False)
    s = tr.compute_grad(None)
    got = {k: p.grad.detach().to(torch.float64).clone() for k, p in tr.policy_net.named_parameters()}
    hs, cs = slot_records(tr, slots)
    rec_h, rec_c = _SlotRecords(hs, tr.args.nagents), _SlotRecords(cs, tr.args.nagents)
    view = _WithRecords(tr, rec_h, rec_c)
    ref, rloss = None, dict.fromkeys(LOSS_KEYS, 0.0)
    for k in slots:
        g, l = trainer_reference(view, slots=(k, k + 1))
        ref = g if ref is None else {q: ref[q] + g[q] for q in ref}
        for q in LOSS_KEYS:
            rloss[q] += l[q]
    abs_sums = slot_heads_abs_sums(tr, rec_h, slots)
    worst = {}
    for k, r in ref.items():
        allowed = TOL * r.abs().max() + (SUM_FLOOR * abs_sums[k] if k in abs_sums else 0.0)
        worst[k] = float(((got[k] - r).abs() / allowed).max()) * TOL
    print("slots %s: %s" % (slots, " ".join("%s %.1e" % kv for kv in worst.items())))
    assert all(v <= TOL for v in worst.values()), worst
    for q in LOSS_KEYS:
        assert np.isclose(s[q], rloss[q], rtol=LOSS_RTOL, atol=LOSS_ATOL), (q, s[q], rloss[q])


# ---------------------------------------------------------------------------------------------------- selection

def test_selection():
    """Default limit: a batch whose records fit keeps full records (before and after the allocation); a limit below
    the full records picks windows; a device too small even for the windows raises an error that names the bytes,
    before anything is allocated for the records, and the trainer stays usable."""
    from ic3net_b200.trainer import Trainer
    tr = make_trainer("grad_pp_hard_ic3net_h128", 400)
    assert tr.record_mode == "full"
    tr.run_batch(0)
    assert tr.record_mode == "full" and "rec_h" in tr._buf
    T = tr._buf["T"]
    need = tr._record_bytes(T)
    tr.RECORD_BYTES_LIMIT = need["full"] - 1
    tr.run_batch(0)                                       # same T: the buffers stay
    assert tr.record_mode == "full"
    tr._alloc(T)
    assert tr.record_mode == "window" and "rec_h" not in tr._buf
    tr.run_batch(0)
    flat_grad(tr)
    tr.RECORD_BYTES_LIMIT = None
    tr.RECORD_MARGIN_BYTES = 1 << 50
    before = torch.cuda.memory_allocated()
    with pytest.raises(RuntimeError, match=r"need [0-9.e+]+ GB for the \(h, c\) records"):
        tr._alloc(T)
    assert torch.cuda.memory_allocated() <= before
    tr.RECORD_MARGIN_BYTES = Trainer.RECORD_MARGIN_BYTES
    tr.run_batch(0)
    assert tr.record_mode == "full"
    flat_grad(tr)
    assert Trainer.RECORD_BYTES_LIMIT is None
