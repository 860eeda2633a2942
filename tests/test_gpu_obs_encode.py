"""GPU tests of the fused observation gather + encoder (ic3_pp_obs_encode / ic3_tj_obs_encode, the dense rollout's
kernels): on live env states, the observation it writes must be exactly what ic3_pp_obs / ic3_tj_obs write, and its x
exactly what the dense encoder computes from that very tensor (and what the index-form encoder computes from the state),
with and without the observation-layout hint, for every supported hid_size."""
import argparse
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import load_golden, ns
from oracle.gen_golden import make_weights

pytestmark = pytest.mark.gpu

CASES = [pytest.param(n, 33, 128, id=n) for n in
         ("env_pp_v1", "env_pp_enemy", "env_pp_comp", "env_pp_hard", "env_tj_medium_v1", "env_tj_hard")]
CASES += [pytest.param("env_pp_hard", 33, h, id="env_pp_hard-H%d" % h) for h in (32, 64)]
CASES += [pytest.param("env_tj_medium_v1", 33, h, id="env_tj_medium_v1-H%d" % h) for h in (32, 64)]
# the full predator-prey hard batch of bench.py (1.19 GB of observations per step)
CASES += [pytest.param("env_pp_hard", 8192, 128, id="env_pp_hard-B8192")]


def _net(nagents, hid, obs_dim):
    from ic3net_b200.comm import CommNetMLP
    heads = (5, 2)
    a = argparse.Namespace(nagents=nagents, hid_size=hid, comm_passes=1, recurrent=True, rnn_type="LSTM",
                           continuous=False, naction_heads=list(heads), comm_mask_zero=False, comm_mode="avg",
                           hard_attn=True, comm_init="uniform", share_weights=False, seed=0, env_id0=0, commnet=True,
                           policy_impl=None)
    net = CommNetMLP(a, obs_dim)
    sd = make_weights(8, obs_dim, hid, heads, "uniform")
    net.load_state_dict({k: torch.from_numpy(v).float() for k, v in sd.items()})
    return net, sd


@pytest.mark.parametrize("hint", [False, True])
@pytest.mark.parametrize("env_name,B,H", CASES)
def test_fused_obs_encoder_equals_gather_then_dense_encoder(env_name, B, H, hint):
    from ic3net_b200 import _lib, data
    meta, _ = load_golden(env_name)
    args = ns(meta["args"], nenvs=B, seed=4, env_id0=0)
    w = data.init(args.env_name, args)
    env = w.env
    is_tj = args.env_name == "traffic_junction"
    NA = args.nagents if is_tj else env.nagent_rows          # agent rows per env (+ the prey with enemy_comm)
    O = w.observation_dim
    net, sd = _net(NA, H, O)
    if hint:
        net.set_obs_layout(*env.obs_layout)
    w.reset(0)
    env.strict = False
    lib = _lib.load()
    obs_fn, enc_fn, idx_fn = ((lib.ic3_tj_obs, lib.ic3_tj_obs_encode, lib.ic3_tj_encoder_index) if is_tj else
                              (lib.ic3_pp_obs, lib.ic3_pp_obs_encode, lib.ic3_pp_encoder_index))
    rs = np.random.RandomState(3)
    big = B > 64
    for t in range(3 if big else 12):
        w.step([rs.randint(0, env.naction, size=(B, NA))])
        cfg = net.policy_cfg(B)
        pk = net.packed()
        s = _lib.stream()
        of = torch.full((B, NA, O), float("nan"), device="cuda")      # every element must be written
        xf = torch.full((B * NA, H), float("nan"), device="cuda")
        _lib.check(enc_fn(C.byref(env.cfg), C.byref(env.state), C.byref(cfg), C.byref(pk), of.data_ptr(), xf.data_ptr(), s))
        og = torch.empty_like(of)
        _lib.check(obs_fn(C.byref(env.cfg), C.byref(env.state), og.data_ptr(), s))
        assert torch.equal(of, og), (env_name, t)
        del og
        xd = torch.empty_like(xf)
        _lib.check(lib.ic3_encoder_dense(C.byref(cfg), C.byref(pk), of.data_ptr(), xd.data_ptr(), s))
        assert torch.equal(xf, xd), (env_name, t)
        xi = torch.empty_like(xf)
        _lib.check(idx_fn(C.byref(env.cfg), C.byref(env.state), C.byref(cfg), C.byref(pk), xi.data_ptr(), s))
        assert torch.equal(xf, xi), (env_name, t)
        # and x is the encoder of the float64 reference on a sample of the rows
        rows = np.sort(rs.choice(B * NA, min(B * NA, 2048), replace=False))
        ref = of.reshape(-1, O)[torch.from_numpy(rows).cuda()].double().cpu().numpy() @ sd["encoder.weight"].T \
            + sd["encoder.bias"]
        got = xf[torch.from_numpy(rows).cuda()].double().cpu().numpy()
        assert np.all(np.abs(got - ref) <= 1e-5 * np.maximum(1.0, np.abs(ref))), (env_name, t)
        del of
    env.err.zero_()

