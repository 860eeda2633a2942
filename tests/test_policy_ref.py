"""CPU tests: the batched float64 policy step of tests/policy_ref.py (the yardstick of tests/test_gpu_policy_rows.py)
against the per-env oracle (oracle/policy.py), against the reference's own forward fixtures, and its Philox draws and
inverse-CDF sampling against oracle/philox.py and oracle.policy.sample_from_logp."""
import numpy as np
import pytest
import torch

from helpers import golden_names, load_golden
from oracle import philox
from oracle import policy as opolicy
from oracle.gen_golden import make_weights
from policy_ref import inverse_cdf, params_f64, philox_u24, step_f64


def same(a, b):
    return np.allclose(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64), rtol=1e-12, atol=1e-13)


def random_sd(rs, O, H, heads, passes, share):
    sd = make_weights(int(rs.randint(1 << 30)), O, H, heads)
    for i in range(1, passes):
        sd["C_modules.%d.weight" % i] = sd["C_modules.0.weight"] if share else rs.uniform(-0.1, 0.1, (H, H))
        sd["C_modules.%d.bias" % i] = sd["C_modules.0.bias"] if share else rs.uniform(-0.1, 0.1, H)
    return sd


# (hard_attn, comm_mode, comm_mask_zero, passes, share_weights)
VARIANTS = [(True, "avg", False, 1, False), (False, "avg", False, 1, False), (True, "sum", False, 1, False),
            (False, "sum", False, 2, False), (True, "avg", True, 1, False), (True, "avg", False, 2, False),
            (True, "avg", False, 3, False), (False, "avg", False, 3, True), (True, "sum", False, 2, True)]


@pytest.mark.parametrize("variant", VARIANTS, ids=["hard%d-%s-zero%d-p%d-share%d" % v for v in VARIANTS])
@pytest.mark.parametrize("N", [1, 2, 3, 10, 32])
def test_step_matches_oracle(N, variant):
    """Envs with no agent alive, exactly one, all of them and a random subset; fresh envs against the oracle fed the
    episode-start inputs (zero state, no comm, everybody alive)."""
    hard, mode, zero, passes, share = variant
    rs = np.random.RandomState(N * 100 + VARIANTS.index(variant))
    B, H, O, heads = 7, 16, 23, (5, 2)
    sd = random_sd(rs, O, H, heads, passes, share)
    P = params_f64(sd, passes)
    roles = opolicy.roles_of(opolicy.params_to_f64(sd), "commnet", True, passes)
    obs = (rs.rand(B, N, O) < 0.2) * rs.randint(1, 4, (B, N, O))
    h, c = rs.uniform(-1, 1, (B, N, H)), rs.uniform(-3, 3, (B, N, H))
    comm, alive = rs.randint(0, 2, (B, N)), rs.randint(0, 2, (B, N))
    alive[0], alive[1], alive[2] = 0, np.eye(1, N, N // 2)[0], 1
    fresh = np.zeros(B, dtype=np.int64)
    fresh[[3, 6]] = 1
    h[3] = np.nan                                   # a fresh env's incoming state is never read
    t = lambda a: torch.as_tensor(a, dtype=torch.float64)
    h2, c2, val, lps = step_f64(P, t(obs.reshape(B * N, O)), t(h.reshape(B * N, H)), t(c.reshape(B * N, H)),
                                t(comm), t(alive), t(fresh), nagents=N, passes=passes, hard_attn=hard, comm_mode=mode,
                                comm_mask_zero=zero)
    h2, c2, val = h2.view(B, N, H).numpy(), c2.view(B, N, H).numpy(), val.view(B, N).numpy()
    for b in range(B):
        if fresh[b]:
            hb, cb, cmb, alb = np.zeros((N, H)), np.zeros((N, H)), np.zeros(N), np.ones(N)
        else:
            hb, cb, cmb, alb = h[b], c[b], comm[b], alive[b].astype(np.float64)
        lo, ov, oh, oc = opolicy.forward_variant(roles, obs[b], hb, cb, cmb if hard else None, alb, hard, mode, zero,
                                                 passes)
        assert same(h2[b], oh) and same(c2[b], oc) and same(val[b], ov), b
        for k in range(len(heads)):
            assert same(lps[k].view(B, N, -1)[b].numpy(), lo[k]), (b, k)


def test_sparse_observation_equals_dense():
    rs = np.random.RandomState(4)
    B, N, H, O, K = 5, 3, 16, 40, 6
    sd = make_weights(9, O, H, (5, 2))
    P = params_f64(sd)
    idx = torch.as_tensor(rs.randint(0, O, (B * N, K)))
    val = torch.as_tensor(rs.randint(0, 3, (B * N, K)), dtype=torch.float64)
    dense = torch.zeros(B * N, O, dtype=torch.float64).index_put_((torch.arange(B * N).repeat_interleave(K),
                                                                  idx.reshape(-1)), val.reshape(-1), accumulate=True)
    h, c = torch.as_tensor(rs.uniform(-1, 1, (2, B * N, H)))
    comm = torch.as_tensor(rs.randint(0, 2, (B, N)))
    a = step_f64(P, (idx, val), h, c, comm, None, None, nagents=N)
    b = step_f64(P, dense, h, c, comm, None, None, nagents=N)
    for x, y in zip(a[:3] + tuple(a[3]), b[:3] + tuple(b[3])):
        assert same(x.numpy(), y.numpy())


@pytest.mark.parametrize("name", golden_names("fwd_"))
def test_step_matches_forward_fixture(name):
    """The reference's own CommNetMLP outputs (float64) for the single-pass variants, all cases as one batch."""
    meta, z = load_golden(name)
    sd = make_weights(meta["weights_seed"], meta["obs_dim"], meta["hid_size"], meta["heads"], meta["comm_init"])
    check_fixture(meta, z, params_f64(sd), 1, meta["hard_attn"], meta["use_alive"], meta["comm_mode"],
                  meta["comm_mask_zero"])


LSTM_VARIANTS = [n for n in golden_names("var_") if load_golden(n)[0]["lstm"]]


@pytest.mark.parametrize("name", LSTM_VARIANTS)
def test_step_matches_variant_fixture(name):
    """The LSTM-cell variant fixtures: comm_passes 2 to 4, share_weights, comm_mode sum, and the RNN (LSTM) baseline of
    models.py, whose C is zero and which never communicates (oracle.policy.roles_of)."""
    meta, z = load_golden(name)
    a = meta["args"]
    sd = {k[3:]: z[k] for k in z.files if k.startswith("sd_")}
    model = meta["model"]
    passes = a["comm_passes"] if model == "commnet" else 1
    hard = bool(meta["hard_attn"]) and model == "commnet"
    check_fixture(meta, z, params_f64(sd, passes, model), passes, hard, meta["use_alive"] and model == "commnet",
                  a["comm_mode"], bool(a["comm_mask_zero"]) or model != "commnet")


def check_fixture(meta, z, P, passes, hard, use_alive, mode, zero):
    K, N, O = z["obs"].shape
    H = z["h"].shape[-1]
    t = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float64)
    h2, c2, val, lps = step_f64(P, t(z["obs"].reshape(K * N, O)), t(z["h"].reshape(K * N, H)),
                                t(z["c"].reshape(K * N, H)), t(z["comm"]) if hard else None,
                                t(z["alive"]) if use_alive else None, None, nagents=N, passes=passes, hard_attn=hard,
                                comm_mode=mode, comm_mask_zero=zero)
    assert same(h2.view(K, N, H).numpy(), z["h2"]) and same(c2.view(K, N, H).numpy(), z["c2"])
    assert same(val.view(K, N).numpy(), z["value"])
    for k in range(len(meta["heads"])):
        assert same(lps[k].view(K, N, -1).numpy(), z["logp%d" % k]), k


def test_philox_u24_matches_oracle():
    rs = np.random.RandomState(5)
    M = 3000
    env = rs.randint(0, 1 << 32, M, dtype=np.uint64)
    env[:10] = np.arange(10)
    tick = rs.randint(0, 1 << 32, M, dtype=np.uint64)
    tick[10:20] = 0
    stream = rs.randint(1, 4, M)
    index = rs.randint(0, 1 << 32, M, dtype=np.uint64)
    index[20:30] = 0xFFFFFFFF
    for seed in (0, 4242, 0xFFFFFFFFFFFFFFFF, int(rs.randint(1 << 62))):
        got = philox_u24(seed, env, tick, stream, index)
        want = np.array([philox.draw_u24(seed, int(e), int(t), int(s), int(i))
                         for e, t, s, i in zip(env, tick, stream, index)])
        assert got.shape == (M, 4) and np.array_equal(got, want), seed
    # broadcasting: one env, a column of ticks, a row of agents
    got = philox_u24(99, 5, np.arange(4)[:, None], philox.STREAM_ACTION, np.arange(3)[None, :])
    assert got.shape == (4, 3, 4)
    assert np.array_equal(got[2, 1], philox.draw_u24(99, 5, 2, philox.STREAM_ACTION, 1))
    assert np.array_equal(got[3, 2, :2], opolicy.action_draws(99, 5, 3, 3, 2)[2])


def test_inverse_cdf_matches_oracle():
    rs = np.random.RandomState(6)
    rows, u24 = [], []
    for na in (1, 2, 3, 5, 16):
        for _ in range(200):
            lp = rs.randn(na) * rs.choice([0.1, 1.0, 5.0])
            rows.append(lp - np.log(np.exp(lp).sum()))
            u24.append(rs.randint(0, 1 << 24))
    for na in (2, 5, 9):                            # hand-built edges
        lp = np.log(np.full(na, 1.0 / na))
        cdf = np.cumsum(np.exp(lp))
        for u in [0, (1 << 24) - 1] + [int(np.floor(v * (1 << 24))) + d for v in cdf[:-1] for d in (-1, 0, 1)]:
            rows.append(lp)
            u24.append(u)
        for extreme in (np.array([0.0] + [-800.0] * (na - 1)), np.array([-800.0] * (na - 1) + [0.0])):
            for u in (0, 1, (1 << 24) - 1):         # a zero-probability action is never drawn
                rows.append(extreme)
                u24.append(u)
    lp = np.array([0.25, 0.25, 0.5])                # a CDF edge exactly on a draw: equal to u is not > u
    rows.append(np.log(lp))
    u24.append(1 << 22)
    for r, u in zip(rows, u24):
        a, m = inverse_cdf(r[None], [u])
        wa, wm = opolicy.sample_from_logp(r, u * 2.0 ** -24)
        assert a[0] == wa and m[0] == wm, (r, u)
    # and as one batch of rows per head size
    for na in (1, 2, 3, 5, 16):
        idx = [k for k, r in enumerate(rows) if len(r) == na]
        a, m = inverse_cdf(np.stack([rows[k] for k in idx]), [u24[k] for k in idx])
        want = [opolicy.sample_from_logp(rows[k], u24[k] * 2.0 ** -24) for k in idx]
        assert np.array_equal(a, [w[0] for w in want]) and np.array_equal(m, [w[1] for w in want])
