"""Worker of tests/test_gpu_graph_update.py: one rank of a 2-GPU NCCL job (launched with torch.distributed.run).
Trains three updates through MultiGPUTrainer, eagerly or with graph_update, and saves what the test compares."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    from helpers import finish_args, load_golden, ns
    from ic3net_b200 import data
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.multi_gpu import MultiGPUTrainer
    from ic3net_b200.trainer import Trainer
    mode, out_dir = sys.argv[1], sys.argv[2]
    rank = int(os.environ["RANK"])
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    meta, _ = load_golden("grad_pp_hard_ic3net_h128")
    B = 12
    args = ns(meta["args"], nenvs=B, seed=808, env_id0=rank * B, obs_mode="index", use_graph=False, policy_impl="tc",
              record_for_grad=True, grad_impl="kernels", graph_update=mode == "graph", lrate=1e-3)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    torch.manual_seed(meta["weights_seed"] + rank)      # different on each rank: rank 0's are broadcast
    net = CommNetMLP(args, args.num_inputs)
    mgt = MultiGPUTrainer(args, lambda: Trainer(args, net, env))
    stats = []
    for ep in range(3):
        s = mgt.train_batch(ep)
        stats.append({k: (v.tolist() if hasattr(v, "tolist") else v) for k, v in s.items()})
    opt = mgt.trainer.optimizer
    torch.save(dict(params=opt.flat_params.cpu(), square_avg=opt.flat_square_avg.cpu(), grads=opt.flat_grads.cpu(),
                    stats=stats), os.path.join(out_dir, "rank%d.pt" % rank))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
