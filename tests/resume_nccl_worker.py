"""Worker of tests/test_gpu_resume.py: one rank of a 2-GPU NCCL job (launched with torch.distributed.run) running
``main.main`` on its arguments with --resumable, where a SIGTERM reaches rank 1 alone during its third update.  The
ranks must agree to stop after that update on both."""
import os
import signal
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from ic3net_b200 import main as m
    from ic3net_b200.multi_gpu import MultiGPUTrainer
    rank = int(os.environ["RANK"])
    orig, calls = MultiGPUTrainer.train_batch, []

    def train_batch(self, epoch):
        calls.append(epoch)
        if rank == 1 and len(calls) == 3:
            signal.raise_signal(signal.SIGTERM)
        return orig(self, epoch)
    MultiGPUTrainer.train_batch = train_batch
    return m.main(sys.argv[1:])


if __name__ == "__main__":
    sys.exit(main())
