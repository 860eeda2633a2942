"""Worker of tests/test_gpu_evaluate.py::test_two_ranks_sum_like_one_process: one rank of a 2-GPU NCCL job (launched
with torch.distributed.run) evaluating on its shard of evaluation slots; dumps the stat dict summed over the ranks."""
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
    args = random_args("c5", nenvs=B, eval_nenvs=B, env_id0=env_id0, max_steps=30)
    return args, make_trainer(args)[1]


def main():
    from ic3net_b200.multi_gpu import MultiGPUTrainer
    out_dir, B = sys.argv[1], int(sys.argv[2])
    rank = int(os.environ["RANK"])
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    args, tr = build(B, rank * B)
    stat = MultiGPUTrainer(args, lambda: tr).evaluate(2)
    np.savez(os.path.join(out_dir, "rank%d.npz" % rank), num_steps=stat["num_steps"],
             num_episodes=stat["num_episodes"], success=stat["success"], reward=np.asarray(stat["reward"]))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
