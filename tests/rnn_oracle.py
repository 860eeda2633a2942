"""Float64 yardstick for the IC / IRIC baselines: models.RNN with the tanh recurrence (rnn_type 'MLP', models.py:59-96)
(TEST INFRASTRUCTURE).

``rnn_oracle()`` is a context in which the float64 oracle (oracle/policy.py, oracle/rollout.py, oracle/grad.py, and the
weights of oracle/gen_golden.py) runs this policy instead of CommNet:
    x = affine1(obs),  h' = tanh(affine2(h) + x),  value_head(h'), log_softmax(heads(h'))        (models.py:81-91)
The value oracle steps through ``oracle.policy.forward_variant`` with the RNN's roles; the gradient oracle restates the
step with torch float64 autograd.  The episode loop, returns, detach cut and loss of oracle/rollout.py and oracle/grad.py
are unchanged: the reference's Trainer drives models.RNN through the same trainer.py code (a zero hidden state at each
episode start, trainer.py:41; detach every detach_gap steps, trainer.py:56-60).  Everything that calls the oracle inside
the context -- ``oracle.gen_golden.gen_grad_case`` writing the ``gradrnn_*`` fixtures from the unmodified reference
(scripts/gen_golden_rnn.py), ``bptt_ref.oracle_grad_sum`` replaying a GPU batch -- then runs the tanh RNN."""
import contextlib

import numpy as np
import torch

from oracle import gen_golden, policy
from oracle import grad as ograd

_make_weights_commnet = gen_golden.make_weights       # captured before any patching


def make_weights(seed, obs_dim, hid, heads, comm_init="uniform"):
    """state_dict of models.RNN (rnn_type 'MLP'): affine1 / affine2 / heads / value_head, drawn by
    oracle.gen_golden.make_weights (the encoder's draw for affine1, the first comm module's for affine2)."""
    sd = _make_weights_commnet(seed, obs_dim, hid, heads, "uniform")
    out = {k: v for k, v in sd.items() if k.startswith("heads.") or k.startswith("value_head.")}
    out.update({"affine1.weight": sd["encoder.weight"], "affine1.bias": sd["encoder.bias"],
                "affine2.weight": sd["C_modules.0.weight"], "affine2.bias": sd["C_modules.0.bias"]})
    return out


def forward_np(params, obs, h, c, comm_action=None, alive=None, hard_attn=True, comm_mode="avg", comm_mask_zero=False):
    """oracle.policy.forward for the tanh RNN: (logps, value, h', c unchanged, x)."""
    roles = policy.roles_of(params, "rnn")
    lo, v, h2, _ = policy.forward_variant(roles, obs, h, None, comm_mask_zero=True)
    x = np.asarray(obs, dtype=np.float64) @ params["affine1.weight"].T + params["affine1.bias"]
    return lo, v, h2, c, x


def forward_torch(p, obs, h, c, comm_action, alive, hard_attn, comm_mode="avg", comm_mask_zero=False):
    """oracle.grad.forward_torch for the tanh RNN (models.py:81-91), differentiable in float64."""
    x = obs @ p["affine1.weight"].t() + p["affine1.bias"]
    h2 = torch.tanh(h @ p["affine2.weight"].t() + p["affine2.bias"] + x)
    value = (h2 @ p["value_head.weight"].t() + p["value_head.bias"])[:, 0]
    logps, k = [], 0
    while "heads.%d.weight" % k in p:
        logps.append(torch.log_softmax(h2 @ p["heads.%d.weight" % k].t() + p["heads.%d.bias" % k], dim=-1))
        k += 1
    return logps, value, h2, c


@contextlib.contextmanager
def rnn_oracle():
    saved = (policy.forward, ograd.forward_torch, gen_golden.make_weights)
    policy.forward, ograd.forward_torch, gen_golden.make_weights = forward_np, forward_torch, make_weights
    try:
        yield
    finally:
        policy.forward, ograd.forward_torch, gen_golden.make_weights = saved
