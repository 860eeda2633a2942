"""Greedy mode of the float64 oracle: every head takes the argmax of its log-probs (the lowest index on a tie, as
torch.argmax), in place of the inverse-CDF draw.  ``with greedy():`` routes oracle.policy.sample_actions, through which
oracle.rollout.run_episode picks its actions, to ``argmax_actions`` for the duration of the block.  TEST
INFRASTRUCTURE, used by scripts/gen_golden_greedy.py and the tests of the tests/golden/greedy_* fixtures."""
import contextlib

import numpy as np

from oracle import policy


def argmax_actions(logps, u24=None):
    """logps: list over heads of [N, na] float64.  Returns (act [N, heads], margin [N, heads]); margin is the gap
    between the two largest log-probs of the head (1.0 for a one-action head): how far the row is from a tie."""
    n = logps[0].shape[0]
    act = np.zeros((n, len(logps)), dtype=np.int64)
    margin = np.ones((n, len(logps)))
    for k, lp in enumerate(logps):
        lp = np.asarray(lp, dtype=np.float64)
        act[:, k] = lp.argmax(-1)
        if lp.shape[-1] > 1:
            top = np.sort(lp, -1)
            margin[:, k] = top[:, -1] - top[:, -2]
    return act, margin


@contextlib.contextmanager
def greedy():
    saved = policy.sample_actions
    policy.sample_actions = argmax_actions
    try:
        yield
    finally:
        policy.sample_actions = saved
