"""GPU tests of the dense rollout on the tensor-core path, where the observation block is written on a side stream while
the policy step runs (Trainer._overlap_obs, ic3_pp_obs_bounded / ic3_tj_obs_bounded): after every lock-step the block
must be exactly what ic3_pp_obs / ic3_tj_obs write for the env state that step's policy consumed, eagerly and inside a
CUDA graph, and at the full predator-prey hard batch, where an env step that moved the
agents before the write had finished would leave wrong cells."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import finish_args, load_golden, ns
from oracle.gen_golden import make_weights

pytestmark = pytest.mark.gpu

BIG_QUOTA = 1 << 30          # no slot halts: every call of _enqueue(1) is one more lock-step of the same rollout


def build(name, B, seed=13, **over):
    from ic3net_b200 import data
    from ic3net_b200.comm import CommNetMLP
    from ic3net_b200.trainer import Trainer
    meta, _ = load_golden(name)
    args = ns(meta["args"], nenvs=B, seed=seed, env_id0=0, obs_mode="dense", policy_impl=None, **over)
    env = data.init(args.env_name, args)
    finish_args(args, env)
    net = CommNetMLP(args, args.num_inputs)
    sd = make_weights(meta["weights_seed"], args.num_inputs, args.hid_size, args.naction_heads, args.comm_init)
    net.load_state_dict({k: torch.from_numpy(v).float() for k, v in sd.items()})
    tr = Trainer(args, net, env)
    tr.OVERLAP_MIN_OBS_BYTES = 0             # the small fixtures take the two-stream path too
    return args, env, tr


CASES = [pytest.param("ep_pp_hard_ic3net", 24, 6, id="pp_hard"),
         pytest.param("ep_pp_enemy_ic3net", 19, 6, id="pp_enemy_comm"),
         pytest.param("ep_tj_medium_ic3net", 16, 6, id="tj_medium"),
         pytest.param("ep_pp_hard_ic3net", 37, 6, id="pp_hard-B37"),
         pytest.param("ep_tj_medium_ic3net", 37, 6, id="tj_medium-B37"),
         pytest.param("ep_pp_hard_ic3net", 8192, 4, id="pp_hard-B8192")]


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name,B,T", CASES)
def test_dense_step_writes_the_observation_its_policy_step_consumed(name, B, T, graph):
    from ic3net_b200 import _lib
    args, env, tr = build(name, B)
    assert tr._overlap_obs()
    e, lib = env.env, _lib.load()
    obs_fn = lib.ic3_tj_obs if tr.is_tj else lib.ic3_pp_obs
    tr._alloc(T)
    tr._episode_boundary(0)
    b = tr._buf
    b["err"].zero_()
    tr.policy_net.packed()
    step = lambda: tr._enqueue(1, quota=BIG_QUOTA)
    step()                                   # eager warm-up step (lazy function attributes)
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        step = g.replay
    obs = b["obs"]
    ref = torch.empty_like(obs)
    locs = []
    for t in range(T):
        locs.append((e.car_loc if tr.is_tj else e.loc).clone())            # positions this step's policy consumes
        _lib.check(obs_fn(C.byref(e.cfg), C.byref(e.state), ref.data_ptr(), _lib.stream()))
        obs.fill_(float("nan"))                                            # every element must be written
        step()
        torch.cuda.synchronize()
        assert torch.equal(obs, ref), (name, t)
    if not tr.is_tj:
        assert all(not torch.equal(p, q) for p, q in zip(locs, locs[1:]))   # the agents moved between the checks
    assert int(b["err"].item()) == 0


def test_small_observation_blocks_keep_the_fused_gather_and_encoder():
    from ic3net_b200.trainer import Trainer
    for B, want in ((24, False), (8192, True)):      # 3.5 MB / 1.19 GB of observations per lock-step
        args, env, tr = build("ep_pp_hard_ic3net", B)
        del tr.OVERLAP_MIN_OBS_BYTES                   # back to the class default
        assert tr.OVERLAP_MIN_OBS_BYTES == Trainer.OVERLAP_MIN_OBS_BYTES
        assert tr._overlap_obs() == want, B


@pytest.mark.parametrize("name", ["ep_pp_hard_ic3net", "ep_tj_medium_ic3net"])
def test_dense_graph_rollout_equals_eager(name):
    """Trainer(use_graph=True) (warm-up on a rewound snapshot, capture, replay) and the eager trainer give the same
    rollout and leave the same observation block, rollout after rollout."""
    res = {}
    for use_graph in (True, False):
        args, env, tr = build(name, 21, seed=5, use_graph=use_graph)
        out = []
        for k in range(2):
            r = tr.rollout(12, 0)
            torch.cuda.synchronize()
            out.append([r.action.cpu().numpy().copy(), r.value.cpu().numpy().copy(), r.reward.cpu().numpy().copy(),
                        tr._buf["obs"].cpu().numpy().copy()])
        res[use_graph] = out
    for a, b in zip(res[True], res[False]):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
