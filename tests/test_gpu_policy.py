"""GPU parity tests of the policy kernels (csrc/policy.cu) through ``CommNetMLP.forward``.
Bar (BASELINE north_star): hidden states / values / log-probs within 1e-5 relative of the
reference CPU path (float64); here |gpu - ref| <= 1e-5 * max(1, |ref|)."""
import argparse

import numpy as np
import pytest
import torch

from gpu_harness import close, cpu
from helpers import finish_args, golden_names, load_golden, make_oracle_env, ns, tj_tables
from oracle import policy as opolicy
from oracle.gen_golden import make_weights

pytestmark = pytest.mark.gpu

IMPLS = ["tc", "simt"]


def build_net(meta_like, nagents, hid, obs_dim, heads, hard_attn, comm_mode="avg", comm_mask_zero=False,
              comm_init="uniform", wseed=0, seed=0, env_id0=0, impl=None):
    if impl == "tc" and hid != 128:
        pytest.skip("tensor-core path is specialised for hid_size 128")
    from ic3net_b200.comm import CommNetMLP
    a = argparse.Namespace(nagents=nagents, hid_size=hid, comm_passes=1, recurrent=True, rnn_type="LSTM",
                           continuous=False, naction_heads=list(heads), comm_mask_zero=comm_mask_zero,
                           comm_mode=comm_mode, hard_attn=hard_attn, comm_init=comm_init, share_weights=False,
                           seed=seed, env_id0=env_id0, commnet=True, policy_impl=impl)
    net = CommNetMLP(a, obs_dim)
    sd = make_weights(wseed, obs_dim, hid, heads, comm_init)
    net.load_state_dict({k: torch.from_numpy(v).float() for k, v in sd.items()})
    return net, a, sd


@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("name", golden_names("fwd_"))
def test_forward_matches_reference_golden(name, impl):
    meta, z = load_golden(name)
    net, a, sd = build_net(meta, meta["nagents"], meta["hid_size"], meta["obs_dim"], meta["heads"],
                           meta["hard_attn"], meta["comm_mode"], meta["comm_mask_zero"], meta["comm_init"],
                           wseed=meta["weights_seed"], impl=impl)
    assert sorted(net.state_dict().keys()) == sorted(sd.keys())      # checkpoint keys interchange
    dev = "cuda"
    for k in range(len(z["obs"])):
        info = {}
        if meta["hard_attn"]:
            info["comm_action"] = z["comm"][k]
        if meta["use_alive"]:
            info["alive_mask"] = z["alive"][k]
        x = [torch.from_numpy(z["obs"][k][None]).float().to(dev),
             (torch.from_numpy(z["h"][k]).float().to(dev), torch.from_numpy(z["c"][k]).float().to(dev))]
        act, val, (h2, c2) = net(x, info)
        assert close(cpu(val)[:, 0], z["value"][k]), name
        assert close(cpu(h2), z["h2"][k]) and close(cpu(c2), z["c2"][k]), name
        for j in range(len(meta["heads"])):
            assert act[j].shape == (1, meta["nagents"], meta["heads"][j])
            assert close(cpu(act[j])[0], z["logp%d" % j][k]), name


@pytest.mark.parametrize("impl", IMPLS)
def test_forward_batched_mixed_masks(impl):
    """B = 77 envs (odd tile tail, envs straddling 128-row tiles), per-env alive / comm masks, vs the float64 oracle."""
    B, N, H, O, heads = 77, 10, 128, 61, (2, 2)
    net, a, sd = build_net(None, N, H, O, heads, True, wseed=3, impl=impl)
    p = opolicy.params_to_f64(sd)
    rs = np.random.RandomState(0)
    obs = (rs.rand(B, N, O) < 0.1) * rs.randint(1, 4, size=(B, N, O))
    h, c = rs.uniform(-1, 1, (B, N, H)), rs.uniform(-2, 2, (B, N, H))
    comm, alive = rs.randint(0, 2, (B, N)), rs.randint(0, 2, (B, N))
    alive[0] = 0
    alive[1] = np.eye(1, N)[0]
    x = [torch.tensor(obs, dtype=torch.float32, device="cuda"),
         (torch.tensor(h.reshape(B * N, H), dtype=torch.float32, device="cuda"),
          torch.tensor(c.reshape(B * N, H), dtype=torch.float32, device="cuda"))]
    act, val, (h2, c2) = net(x, {"comm_action": comm, "alive_mask": alive.astype(np.float64)})
    val, h2, c2 = cpu(val).reshape(B, N), cpu(h2).reshape(B, N, H), cpu(c2).reshape(B, N, H)
    for b in range(B):
        lo, ov, oh, oc, _ = opolicy.forward(p, obs[b], h[b], c[b], comm[b], alive[b].astype(float), True)
        assert close(val[b], ov) and close(h2[b], oh) and close(c2[b], oc), b
        for j in range(2):
            assert close(cpu(act[j])[b], lo[j]), b


@pytest.mark.parametrize("H,N,O,heads", [(32, 3, 29, (5, 2)), (64, 5, 45, (5,)), (128, 20, 149, (2, 2)),
                                          (128, 32, 40, (3, 4, 2))])
@pytest.mark.parametrize("impl", IMPLS)
def test_forward_shapes(H, N, O, heads, impl):
    B = 13
    net, a, sd = build_net(None, N, H, O, heads, len(heads) > 1, wseed=H + N, impl=impl)
    p = opolicy.params_to_f64(sd)
    rs = np.random.RandomState(1)
    obs = rs.uniform(-1, 1, (B, N, O)) * (rs.rand(B, N, O) < 0.3)
    h, c = rs.uniform(-1, 1, (B, N, H)), rs.uniform(-1, 1, (B, N, H))
    comm = rs.randint(0, 2, (B, N))
    x = [torch.tensor(obs, dtype=torch.float32, device="cuda"),
         (torch.tensor(h.reshape(-1, H), dtype=torch.float32, device="cuda"),
          torch.tensor(c.reshape(-1, H), dtype=torch.float32, device="cuda"))]
    act, val, (h2, c2) = net(x, {"comm_action": comm})
    for b in range(B):
        lo, ov, oh, oc, _ = opolicy.forward(p, obs[b], h[b], c[b], comm[b] if len(heads) > 1 else None, None,
                                            len(heads) > 1)
        assert close(cpu(h2).reshape(B, N, H)[b], oh) and close(cpu(c2).reshape(B, N, H)[b], oc)
        assert close(cpu(val).reshape(B, N)[b], ov)
        for j in range(len(heads)):
            assert close(cpu(act[j])[b], lo[j])


def test_select_action_inverse_cdf():
    """select_action on explicit draws == oracle inverse CDF (where fp32 cannot flip the draw)."""
    from ic3net_b200.action_utils import select_action
    B, N, heads = 50, 10, (5, 2)
    rs = np.random.RandomState(2)
    logits = [rs.randn(B, N, na) for na in heads]
    logp = [l - np.log(np.exp(l).sum(-1, keepdims=True)) for l in logits]
    u24 = rs.randint(0, 1 << 24, size=(B, N, len(heads)))
    a = argparse.Namespace(continuous=False, seed=0)
    act = cpu(select_action(a, [torch.tensor(l, dtype=torch.float32, device="cuda") for l in logp], draws=u24))
    for b in range(B):
        want, margin = opolicy.sample_actions([l[b] for l in logp], u24[b])
        ok = margin > 1e-5
        assert np.array_equal(act[b][ok], want[ok])
    # Philox action stream: same draws as the oracle's stream
    tick = torch.full((B,), 17, dtype=torch.int32, device="cuda")
    a.seed, a.env_id0 = 99, 5
    act = cpu(select_action(a, [torch.tensor(l, dtype=torch.float32, device="cuda") for l in logp], tick=tick))
    for b in range(0, B, 7):
        d = opolicy.action_draws(99, 5 + b, 17, N, len(heads))
        want, margin = opolicy.sample_actions([l[b] for l in logp], d)
        ok = margin > 1e-5
        assert np.array_equal(act[b][ok], want[ok])


@pytest.mark.parametrize("hint", [False, True])
@pytest.mark.parametrize("env_name", ["env_pp_v1", "env_pp_hard", "env_tj_medium_v1", "env_tj_hard"])
def test_index_encoder_equals_dense_encoder(env_name, hint):
    """x from the env state (no obs tensor) must be bit-identical to x = encoder(obs), with and without the
    observation-layout hint (class terms and counts summed separately); the per-position table of the class
    terms must be exactly what those kernels add up."""
    import ctypes as C
    from ic3net_b200 import _lib, data
    meta, z = load_golden(env_name)
    B = 33
    args = ns(meta["args"], nenvs=B, seed=4, env_id0=0)
    w = data.init(args.env_name, args)
    env = w.env
    is_tj = args.env_name == "traffic_junction"
    O = w.observation_dim
    net, a, sd = build_net(None, args.nagents, 128, O, (5, 2), True, wseed=8)
    if hint:
        net.set_obs_layout(*env.obs_layout)
    obs = w.reset(0)
    env.strict = False
    rs = np.random.RandomState(3)
    lib = _lib.load()
    for t in range(12):
        obs, r, done, info = w.step([rs.randint(0, env.naction, size=(B, args.nagents))])
        cfg = net.policy_cfg(B)
        pk = net.packed()
        xd = torch.empty(B * args.nagents, 128, device="cuda")
        xi = torch.empty_like(xd)
        _lib.check(lib.ic3_encoder_dense(C.byref(cfg), C.byref(pk), obs.contiguous().data_ptr(), xd.data_ptr(),
                                         _lib.stream()))
        if is_tj:
            _lib.check(lib.ic3_tj_encoder_index(C.byref(env.cfg), C.byref(env.state), C.byref(cfg), C.byref(pk),
                                                xi.data_ptr(), _lib.stream()))
        else:
            _lib.check(lib.ic3_pp_encoder_index(C.byref(env.cfg), C.byref(env.state), C.byref(cfg), C.byref(pk),
                                                xi.data_ptr(), _lib.stream()))
        assert torch.equal(xd, xi), (env_name, t)
        ref = cpu(obs).reshape(-1, O).astype(np.float64) @ sd["encoder.weight"].T + sd["encoder.bias"]
        assert close(cpu(xd), ref)
    if hint:
        # table[pos] = bias + class terms of an agent standing at pos: check against float64, and against the
        # dense encoder on an observation that holds only class features (exactly the same additions)
        tab = torch.empty(env.obs_positions, 128, device="cuda")
        fn = lib.ic3_tj_encoder_table if is_tj else lib.ic3_pp_encoder_table
        _lib.check(fn(C.byref(env.cfg), C.byref(cfg), C.byref(pk), tab.data_ptr(), _lib.stream()))
        off, V, ncount = env.obs_layout
        o = cpu(obs).reshape(-1, O).copy()
        cells = o[:, off:].reshape(o.shape[0], -1, V)
        cells[:, :, V - ncount:] = 0                      # drop the counts ...
        o[:, :off] = 0                                    # ... and the scalars
        loc = cpu(env.car_loc if is_tj else env.loc)
        alive = cpu(env.alive_mask) if is_tj else None
        rows, want64 = [], []
        for b_ in range(B):
            for i in range(args.nagents):
                if is_tj and not alive[b_, i]:
                    continue                              # dead cars have an all-zero observation
                r_, c_ = loc[b_, i]
                rows.append(b_ * args.nagents + i)
                want64.append(int(r_) * (env.dims[1] if is_tj else env.dim) + int(c_))
        if rows:
            od = torch.from_numpy(o).float().cuda().reshape(B, args.nagents, O).contiguous()
            xc = torch.empty(B * args.nagents, 128, device="cuda")
            _lib.check(lib.ic3_encoder_dense(C.byref(cfg), C.byref(pk), od.data_ptr(), xc.data_ptr(), _lib.stream()))
            assert torch.equal(xc[rows], tab[want64])
            ref = o[rows].astype(np.float64) @ sd["encoder.weight"].T + sd["encoder.bias"]
            assert close(cpu(tab[want64]), ref)
    env.err.zero_()
