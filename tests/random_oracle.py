"""Float64 yardstick for the Random baseline (models.Random, models.py:37-56) on the trainer's non-recurrent branch
(trainer.py:61-65) (TEST INFRASTRUCTURE).

Random.forward ignores the observation apart from its shape and returns value = torch.rand(..., 1) and, per action head,
log_softmax(torch.randn(..., na)).  Here those draws come from Philox stream 4 (oracle/philox.py), the stream the CUDA
step ic3_random_policy_step (ic3net_b200/csrc/random_policy.cu) reads:

    stream 4  Random policy   tick = env step counter (the action stream's tick), index = 4 * agent + block;
                              agent i's words u[0..15] are the four words of blocks 0..3 in order
    value    = u[0] * 2**-24
    logit j  = sqrt(-2 ln((u[1 + 2j] + 1) * 2**-24)) * cos(2 pi u[2 + 2j] * 2**-24)     (heads concatenated)

Actions are then sampled like every other policy (action stream 3, inverse CDF: oracle/policy.py).  ``run_episode`` is
Trainer.get_episode for this policy (no hidden state, no communication) and ``losses`` the three sums of compute_grad
(trainer.py:128-225), which reach no parameter."""
import numpy as np

from oracle import philox, policy
from oracle.grad import returns_np

STREAM_RANDOM_POLICY = 4
RANDOM_WORDS = 16


def _draw24(seed, env_ids, ticks, stream, index):
    """24-bit words [..., 4] of the counters (env_ids, ticks, stream, index), broadcast against each other."""
    env_ids, ticks, index = np.broadcast_arrays(*(np.asarray(a, dtype=np.uint64) for a in (env_ids, ticks, index)))
    ctr = np.stack([env_ids, ticks, np.full_like(env_ids, stream), index], -1)
    return (philox.philox4x32(ctr, philox.split_seed(seed)) >> np.uint32(8)).astype(np.int64)


def words(seed, env_ids, ticks, agents):
    """u[..., 0:16]: the stream-4 words of agent rows (env_ids, ticks, agents), broadcast against each other."""
    agents = np.asarray(agents, dtype=np.uint64)
    return np.concatenate([_draw24(seed, env_ids, ticks, STREAM_RANDOM_POLICY, 4 * agents + b)
                           for b in range(RANDOM_WORDS // 4)], -1)


def action_words(seed, env_ids, ticks, agents, nheads):
    """Action-stream words [..., nheads] of agent rows (oracle/policy.py action_draws over whole arrays)."""
    return _draw24(seed, env_ids, ticks, philox.STREAM_ACTION, agents)[..., :nheads]


def value_logits(u, atot):
    """(value [...], logits [..., atot]) of agent rows from their stream-4 words u [..., 16] (float64)."""
    u = np.asarray(u, dtype=np.int64)
    j = np.arange(atot)
    u1, u2 = u[..., 1 + 2 * j].astype(np.float64), u[..., 2 + 2 * j].astype(np.float64)
    z = np.sqrt(-2.0 * np.log((u1 + 1.0) * 2.0 ** -24)) * np.cos(np.pi * u2 * 2.0 ** -23)
    return u[..., 0] * 2.0 ** -24, z


def step(heads, u, act_u24):
    """Random.forward + select_action on agent rows.  heads: action head sizes; u [R, 16] stream-4 words; act_u24
    [R, nheads] action-stream words.  Returns (value [R], log-probs per head [R, na], act [R, nheads], margin [R,
    nheads]: distance of the action draw to the nearest inner CDF edge, oracle/policy.py sample_from_logp)."""
    value, logits = value_logits(u, int(sum(heads)))
    offs = np.concatenate([[0], np.cumsum(heads)]).astype(int)
    logps = [policy._log_softmax(logits[:, offs[k]:offs[k + 1]]) for k in range(len(heads))]
    act = np.zeros((len(value), len(heads)), dtype=np.int64)
    margin = np.ones((len(value), len(heads)))
    for k, lp in enumerate(logps):
        cdf = np.cumsum(np.exp(lp), -1)
        uu = act_u24[:, k:k + 1] * 2.0 ** -24
        hit = cdf > uu
        act[:, k] = np.where(hit.any(-1), hit.argmax(-1), lp.shape[1] - 1)
        if lp.shape[1] > 1:
            margin[:, k] = np.abs(cdf[:, :-1] - uu).min(-1)
    return value, logps, act, margin


def run_episode(env, args, seed, env_id, epoch=0, tick0=0, episode=0):
    """Trainer.get_episode (trainer.py:26-126) with models.Random for ONE environment (oracle/rollout.py without the
    observation, hidden state and communication Random does not read)."""
    n, heads = args.nagents, list(args.naction_heads)
    is_tj = args.env_name == "traffic_junction"
    if is_tj:
        env.tick = tick0
        env.reset(epoch)
    else:
        env.reset(seed=seed, env_id=env_id, episode=episode)
    rec = dict(act=[], reward=[], value=[], alive=[], mini=[], emask=[], margin=[], logp=[], loc=[])
    for t in range(args.max_steps):
        i = np.arange(n)
        v, lo, a, margin = step(heads, words(seed, env_id, tick0 + t, i),
                                action_words(seed, env_id, tick0 + t, i, len(heads)))
        if is_tj:
            _, rew, done, info = env.step(a[:, 0], seed=seed, env_id=env_id)
            alive = info["alive_mask"]
            loc = env.car_loc.copy()
        else:
            _, rew, done, info = env.step(a[:, 0])
            alive = np.ones(n)
            loc = np.concatenate([env.predator_loc, env.prey_loc]).copy()
        done = bool(done) or t == args.max_steps - 1
        mini = np.ones(n)
        if not done and is_tj:
            mini = 1 - info["is_completed"]
        if done:
            rew = rew + env.reward_terminal()
        rec["act"].append(a); rec["reward"].append(rew); rec["value"].append(v); rec["alive"].append(alive.copy())
        rec["mini"].append(mini); rec["emask"].append(np.zeros(n) if done else np.ones(n)); rec["margin"].append(margin)
        rec["logp"].append(np.concatenate(lo, axis=-1)); rec["loc"].append(loc)
        if done:
            break
    out = {k: np.array(v) for k, v in rec.items()}
    out["success"] = int(env.stat.get("success", -1))
    out["num_steps"] = len(rec["act"])
    return out


def run_batch(env, args, seed, env_id, epoch=0):
    """Trainer.run_batch (trainer.py:227-242) of one env slot: whole episodes until >= batch_size steps."""
    eps, tick = [], 0
    while tick < args.batch_size:
        ep = run_episode(env, args, seed, env_id, epoch, tick0=tick, episode=len(eps))
        eps.append(ep)
        tick += ep["num_steps"]
    return eps


def losses(episodes, args):
    """compute_grad's action_loss, value_loss and entropy (trainer.py:160-220) of one slot's batch, float64; returns
    (loss dict, returns [T, N])."""
    cat = lambda k: np.concatenate([ep[k] for ep in episodes])
    heads = list(args.naction_heads)
    offs = np.concatenate([[0], np.cumsum(heads)])
    value, logp, act, alive = cat("value"), cat("logp"), cat("act"), cat("alive")
    ret = returns_np(cat("reward"), cat("emask"), cat("mini"), args.gamma, args.mean_ratio)
    adv = ret - value
    if args.normalize_rewards:
        adv = (adv - adv.mean()) / adv.std(ddof=1)
    lp = sum(np.take_along_axis(logp[..., offs[k]:offs[k + 1]], act[..., k:k + 1], -1)[..., 0]
             for k in range(len(heads)))
    return dict(action_loss=float((-adv * lp * alive).sum()), value_loss=float(((value - ret) ** 2 * alive).sum()),
                entropy=float(-(logp * np.exp(logp)).sum())), ret
