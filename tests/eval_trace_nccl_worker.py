"""Worker of tests/test_gpu_eval_trace.py::test_two_ranks_equal_one_process: one rank of a 2-GPU NCCL job (launched
with torch.distributed.run) recording an evaluation of its shard of evaluation slots; dumps the stat summed over the
ranks, the comm map summed over the ranks and this rank's trace."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def build(B, env_id0):
    from gpu_harness import PP, update_trainer
    return None, update_trainer(PP, B, False, eval_nenvs=B, env_id0=env_id0, max_steps=30, record_for_grad=False)


def main():
    from ic3net_b200.multi_gpu import MultiGPUTrainer
    out_dir, B = sys.argv[1], int(sys.argv[2])
    rank = int(os.environ["RANK"])
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    _, tr = build(B, rank * B)
    stat, trace, cmap = MultiGPUTrainer(tr.args, lambda: tr).evaluate_trace(2, slots=B)
    out = dict(num_steps=stat["num_steps"], num_episodes=stat["num_episodes"], **trace.arrays())
    out.update({"map_" + k: v for k, v in cmap.items()})
    np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **out)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
