"""Worker of tests/test_gpu_random.py::test_two_ranks_reduce_like_one_process: one rank of a 2-GPU NCCL job (launched
with torch.distributed.run) training the Random baseline on its shard of env slots; dumps the reduced statistics."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def build(B, env_id0):
    from gpu_harness import random_args, random_trainer as make_trainer
    args = random_args("c5", nenvs=B, env_id0=env_id0, batch_size=100, gamma=0.9, normalize_rewards=True, entr=0.01)
    return args, make_trainer(args)[1]


def main():
    from ic3net_b200.multi_gpu import MultiGPUTrainer
    out_dir, B = sys.argv[1], int(sys.argv[2])
    rank = int(os.environ["RANK"])
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    args, tr = build(B, rank * B)
    stat = MultiGPUTrainer(args, lambda: tr).train_batch(0)
    np.savez(os.path.join(out_dir, "rank%d.npz" % rank), num_steps=stat["num_steps"],
             num_episodes=stat["num_episodes"], success=stat["success"], reward=np.asarray(stat["reward"]),
             losses=np.array([stat[k] for k in ("action_loss", "value_loss", "entropy")]),
             params=tr.optimizer.flat_params.cpu().numpy())
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
