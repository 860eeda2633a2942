"""GPU tests of resuming a run (main.py --resumable / --resume, Trainer.run_state / load_run_state).

Each case runs main.main in this process three times, each on a fresh trainer: an uninterrupted run of E epochs, the
same run stopped after k epochs (or by a signal), and a --resume of the stopped run up to E epochs.  The final
checkpoints (parameters, RMSprop state, log, evaluation results), the run-state sidecars and the printed Epoch / Eval
lines without their timings must be bit-identical between the uninterrupted and the resumed run."""
import os
import re
import signal
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

from gpu_harness import LOSS_ATOL, LOSS_RTOL, ROOT, TOL

pytestmark = pytest.mark.gpu

PP = ["--env_name", "predator_prey", "--nagents", "3", "--dim", "5", "--vision", "1", "--max_steps", "20", "--mode",
      "mixed", "--hid_size", "128", "--nenvs", "16", "--epoch_size", "2", "--batch_size", "30", "--detach_gap", "10",
      "--lrate", "0.001"]
IC3 = ["--ic3net", "--recurrent"]
# add_rate moves at epochs 1, 2 and 3: a stop after 2 epochs falls inside the curriculum window
TJ = ["--env_name", "traffic_junction", "--nagents", "5", "--dim", "6", "--vision", "0", "--max_steps", "20",
      "--hid_size", "128", "--ic3net", "--recurrent", "--nenvs", "16", "--epoch_size", "2", "--batch_size", "20",
      "--difficulty", "easy", "--add_rate_min", "0.1", "--add_rate_max", "0.3", "--curr_start", "1", "--curr_end", "4",
      "--lrate", "0.001", "--seed", "5"]
RESULT_LINES = ("Epoch ", "Enemy-Reward:", "Add-Rate:", "Success:", "Steps-taken:", "Comm-Action:", "Enemy-Comm:",
                "Eval ")


def result_lines(out):
    """The Epoch / Eval lines of a run's output, without the epoch time."""
    return [re.sub(r"\tTime [0-9.]+s", "", ln) for ln in out.splitlines() if ln.startswith(RESULT_LINES)]


def run_main(argv, capsys):
    from ic3net_b200 import main as m
    capsys.readouterr()
    assert m.main(argv) == 0
    return result_lines(capsys.readouterr().out)


def load(path):
    from ic3net_b200 import main as m
    with m._utils_alias():
        return torch.load(path, weights_only=False)


def assert_same(a, b, where="file"):
    """Bit equality of nested checkpoint / sidecar contents."""
    assert type(a) is type(b), (where, type(a), type(b))
    if isinstance(a, dict):
        assert sorted(a, key=str) == sorted(b, key=str), (where, sorted(a, key=str), sorted(b, key=str))
        for k in a:
            assert_same(a[k], b[k], "%s[%r]" % (where, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), (where, len(a), len(b))
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, "%s[%d]" % (where, i))
    elif torch.is_tensor(a):
        assert a.dtype == b.dtype and torch.equal(a, b), where
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and np.array_equal(a, b), where
    else:
        assert a == b, (where, a, b)


def assert_same_run(a, b):
    assert_same(load(a), load(b), "checkpoint")
    assert_same(load(a + ".run"), load(b + ".run"), "run state")


def stop_and_resume(tmp_path, capsys, argv, E, k, between=None, full="full.pt"):
    """Uninterrupted E epochs into tmp_path/full, k epochs into tmp_path/part, then --resume of part up to E; returns
    (printed lines of the uninterrupted run, of the stopped and resumed runs, the two checkpoint paths)."""
    full, part = str(tmp_path / full), str(tmp_path / "part.pt")
    want = run_main(argv + ["--num_epochs", str(E), "--resumable", "--save", full], capsys)
    got = run_main(argv + ["--num_epochs", str(k), "--resumable", "--save", part], capsys)
    assert (load(part + ".run")["ep"], load(part + ".run")["update"]) == (k, 0)
    if between is not None:
        between()
    got += run_main(argv + ["--num_epochs", str(E), "--resume", part, "--save", part], capsys)
    assert len([ln for ln in want if ln.startswith("Epoch ")]) == E
    return want, got, full, part


CASES = {
    "ic3net_tc": (PP + IC3 + ["--seed", "4"], 3, 1),
    "ic3net_use_graph": (PP + IC3 + ["--seed", "4", "--use_graph"], 3, 1),
    "ic3net_graph_update": (PP + IC3 + ["--seed", "4", "--graph_update"], 3, 2),
    "ic3net_windows": (PP + IC3 + ["--seed", "6"], 3, 1),
    "ic_tc_tanh": (PP + ["--recurrent", "--policy_impl", "tc_tanh", "--grad_impl", "kernels", "--seed", "4"], 3, 1),
    "random": (PP + ["--random", "--seed", "4"], 3, 1),
    "enemy_comm": (PP + IC3 + ["--enemy_comm", "--seed", "7"], 3, 1),
    "eval_sampled": (PP + IC3 + ["--seed", "4", "--eval_every", "1", "--eval_nenvs", "8"], 3, 1),
    "tj_curriculum": (TJ, 5, 2),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_resumed_run_equals_uninterrupted(tmp_path, capsys, monkeypatch, case):
    from ic3net_b200.trainer import Trainer
    argv, E, k = CASES[case]
    if case == "ic3net_windows":
        monkeypatch.setattr(Trainer, "RECORD_BYTES_LIMIT", 0)      # full records never fit: window records
    want, got, full, part = stop_and_resume(tmp_path, capsys, argv, E, k)
    assert got == want
    assert_same_run(full, part)
    run = load(part + ".run")
    if case == "eval_sampled":
        # the evaluation env's streams moved on before the stop, and the resumed evaluations continued them
        assert int(load(str(tmp_path / "full.pt") + ".run")["state"]["ranks"][0]["eval"]["device"]["tick"].sum()) > 0
        assert len([ln for ln in want if ln.startswith("Eval ")]) == E and len(load(full)["eval"]) == E
    if case == "tj_curriculum":
        rates = [ln for ln in want if ln.startswith("Add-Rate:")]
        assert len(set(rates)) >= 3, rates                            # add_rate moved before and after the stop
        assert run["state"]["ranks"][0]["env"]["add_rate"] > 0.1


def test_kernels_ff_resume_keeps_the_recorded_chunk_length(tmp_path, capsys, monkeypatch):
    """models.MLP with kernels_ff: the resumed run takes the chunk length K of the stopped run's last update, even when
    a different FF_CHUNK_ROWS cap (K = 1 here) would measure another one."""
    from ic3net_b200.trainer import Trainer
    argv = PP + ["--policy_impl", "tc_ff", "--grad_impl", "kernels_ff", "--seed", "4"]
    want, got, full, part = stop_and_resume(tmp_path, capsys, argv, 3, 1,
                                            between=lambda: monkeypatch.setattr(Trainer, "FF_CHUNK_ROWS", 16 * 3))
    K = load(full + ".run")["state"]["ranks"][0]["ff_chunk_steps"]
    assert K > 1
    assert got == want
    assert_same_run(full, part)


def test_seed_minus_one_resumes_on_the_stored_seed(tmp_path, capsys):
    from ic3net_b200 import main as m
    argv = PP + IC3 + ["--seed", "-1"]
    part = str(tmp_path / "part.pt")
    got = run_main(argv + ["--num_epochs", "1", "--resumable", "--save", part], capsys)
    seed = load(part + ".run")["state"]["fingerprint"]["seed"]
    assert seed >= 0
    full = str(tmp_path / "full.pt")
    want = run_main(PP + IC3 + ["--seed", str(seed), "--num_epochs", "3", "--resumable", "--save", full], capsys)
    with pytest.raises(ValueError, match="seed \\(stored %d, now %d\\)" % (seed, seed + 1)):
        m.main(PP + IC3 + ["--seed", str(seed + 1), "--num_epochs", "3", "--resume", part, "--save", part])
    got += run_main(argv + ["--num_epochs", "3", "--resume", part, "--save", part], capsys)
    assert got == want
    assert_same_run(full, part)


def test_autograd_resume(tmp_path, capsys, record_property):
    """grad_impl autograd: bit equality if two uninterrupted runs agree bit for bit, the autograd bar otherwise."""
    argv = PP + IC3 + ["--seed", "4", "--grad_impl", "autograd"]
    again = str(tmp_path / "again.pt")
    twice = run_main(argv + ["--num_epochs", "3", "--resumable", "--save", again], capsys)
    want, got, full, part = stop_and_resume(tmp_path, capsys, argv, 3, 1)
    try:
        assert_same_run(full, again)
        deterministic = twice == want
    except AssertionError:
        deterministic = False
    record_property("autograd_bar", "bit equality" if deterministic else "tolerance")
    print("autograd resume compared by", "bit equality" if deterministic else "the autograd tolerance")
    if deterministic:
        assert got == want
        assert_same_run(full, part)
        return
    a, b = load(full), load(part)
    for key, w in a["policy_net"].items():
        err = float((b["policy_net"][key] - w).abs().max())
        assert err <= TOL * max(float(w.abs().max()), 1e-30), (key, err)
    for name in ("reward", "value_loss", "action_loss", "entropy"):
        assert np.allclose(np.asarray(b["log"][name].data, dtype=np.float64),
                           np.asarray(a["log"][name].data, dtype=np.float64), rtol=LOSS_RTOL, atol=LOSS_ATOL), name


def test_stop_by_signal_mid_epoch_in_process(tmp_path, capsys, monkeypatch):
    """SIGTERM during the third update (epoch 2 of 2-update epochs): the run saves after that update and returns 0,
    and the resume from the middle of epoch 2 equals the uninterrupted run."""
    from ic3net_b200.multi_gpu import MultiGPUTrainer
    argv = PP + IC3 + ["--seed", "4", "--num_epochs", "3"]
    full, part = str(tmp_path / "full.pt"), str(tmp_path / "part.pt")
    want = run_main(argv + ["--resumable", "--save", full], capsys)
    orig, calls = MultiGPUTrainer.train_batch, []

    def train_batch(self, epoch):
        calls.append(epoch)
        if len(calls) == 3:
            signal.raise_signal(signal.SIGTERM)
        return orig(self, epoch)
    monkeypatch.setattr(MultiGPUTrainer, "train_batch", train_batch)
    capsys.readouterr()
    from ic3net_b200 import main as m
    handlers = [signal.getsignal(s) for s in (signal.SIGTERM, signal.SIGINT)]
    assert m.main(argv + ["--resumable", "--save", part]) == 0
    out = capsys.readouterr().out
    assert "Stopped in epoch 2 after update 1 of 2; continue with --resume " + part in out
    assert len(calls) == 3 and [signal.getsignal(s) for s in (signal.SIGTERM, signal.SIGINT)] == handlers
    run = load(part + ".run")
    assert (run["ep"], run["update"], run["steps"], run["epochs"]) == (1, 1, 3, 1) and run["stat"]["num_steps"] > 0
    monkeypatch.setattr(MultiGPUTrainer, "train_batch", orig)
    got = result_lines(out) + run_main(argv + ["--resume", part, "--save", part], capsys)
    assert got == want
    assert_same_run(full, part)


def test_stop_by_sigterm_subprocess(tmp_path, capsys):
    """python -m ic3net_b200.main --resumable, sent SIGTERM once its first Epoch line appears, exits 0 after the update in
    flight; its resume equals the uninterrupted run."""
    argv = PP + IC3 + ["--seed", "4", "--epoch_size", "4", "--num_epochs", "25"]
    part = str(tmp_path / "part.pt")
    p = subprocess.Popen([sys.executable, "-u", "-m", "ic3net_b200.main"] + argv + ["--resumable", "--save", part],
                         cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    watchdog = threading.Timer(600, p.kill)
    watchdog.start()
    try:
        out = []
        for line in p.stdout:
            out.append(line)
            if line.startswith("Epoch "):
                p.send_signal(signal.SIGTERM)
                break
        out.append(p.stdout.read())               # through the same buffered reader: nothing read ahead is lost
        p.wait(timeout=600)
        out = "".join(out)
        assert p.returncode == 0, out[-4000:]
    finally:
        watchdog.cancel()
        if p.poll() is None:
            p.kill()
        p.wait(timeout=60)
    assert "Stopped in epoch " in out, out[-4000:]
    run = load(part + ".run")
    assert run["ep"] * 4 + run["update"] < 25 * 4
    print("stopped at epoch index %d, update %d" % (run["ep"], run["update"]))
    got = result_lines(out) + run_main(argv + ["--resume", part, "--save", part], capsys)
    full = str(tmp_path / "full.pt")
    want = run_main(argv + ["--resumable", "--save", full], capsys)
    assert got == want
    assert_same_run(full, part)


def test_refusals(tmp_path, capsys):
    from ic3net_b200 import main as m
    argv = PP + IC3 + ["--seed", "4"]
    a, b = str(tmp_path / "a.pt"), str(tmp_path / "b.pt")
    run_main(argv + ["--num_epochs", "1", "--resumable", "--save", a], capsys)
    run_main(argv + ["--num_epochs", "2", "--resumable", "--save", b], capsys)
    with pytest.raises(ValueError, match=r"nenvs \(stored 16, now 8\)"):
        m.main([x if x != "16" else "8" for x in argv] + ["--num_epochs", "3", "--resume", a, "--save", a])
    with pytest.raises(ValueError, match=r"use_graph \(stored False, now True\)"):
        m.main(argv + ["--use_graph", "--num_epochs", "3", "--resume", a])
    with pytest.raises(ValueError, match=r"batch_size \(stored 30, now 40\)"):
        m.main([x if x != "30" else "40" for x in argv] + ["--num_epochs", "3", "--resume", a])
    os.replace(a + ".run", b + ".run")                   # b's checkpoint beside a's sidecar
    with pytest.raises(ValueError, match="does not belong"):
        m.main(argv + ["--num_epochs", "3", "--resume", b])
    with pytest.raises(FileNotFoundError, match="--resumable"):
        m.main(argv + ["--num_epochs", "3", "--resume", a])
    for extra, message in ((["--resume", b, "--load", b], "takes no --load"), (["--resumable"], "give --save")):
        with pytest.raises(SystemExit):
            m.main(argv + ["--num_epochs", "3"] + extra)
        assert message in capsys.readouterr().err


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_stop_and_resume(tmp_path):
    """Two ranks under NCCL: rank 1 alone is signalled during its third update; both ranks stop after it, and the
    resume equals the uninterrupted two-rank run."""
    argv = PP + IC3 + ["--seed", "4", "--num_epochs", "3"]
    full, part = str(tmp_path / "full.pt"), str(tmp_path / "part.pt")
    worker = os.path.join(ROOT, "tests", "resume_nccl_worker.py")

    def launch(port, target, extra):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
               "127.0.0.1", "--master-port", str(port)] + target + argv + extra
        r = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-4000:]
        return r.stdout
    want = result_lines(launch(29781, ["-m", "ic3net_b200.main"], ["--resumable", "--save", full]))
    out = launch(29782, [worker], ["--resumable", "--save", part])
    assert "Stopped in epoch 2 after update 1 of 2" in out
    got = result_lines(out) + result_lines(launch(29783, ["-m", "ic3net_b200.main"], ["--resume", part, "--save", part]))
    assert got == want
    assert_same_run(full, part)
    assert len(load(part + ".run")["state"]["ranks"]) == 2
