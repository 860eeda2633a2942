"""Traffic junction with ``vocab_type='scalar'`` on the CPU (TEST INFRASTRUCTURE).

``TrafficJunctionScalarOracle`` is oracle/tj_env.py's ``TrafficJunctionOracle`` with the scalar vocabulary of the
reference's ``ic3net_envs/traffic_junction_env.py``:
  multi_agent_init :139-148  vocab_size 2 (road, car), OUTSIDE 0 / ROAD 1 / CAR 2 with no BASE offset, and a
                             MultiDiscrete(dims) member in the observation space: observation_dim = 4 + W*W*2
  _set_grid        :300-314  road-class grid, no per-cell numbering
  _get_obs         :321-366  window one-hot with vocab_size + 1 columns whose OUTSIDE column is dropped (:331-332):
                             per cell (is_road, car count incl. dead cars at (0,0)); per car
                             (last_act/(naction-1), route_id/(npath-1), loc/(h-1, w-1), window), all zero when dead
Dynamics, rewards, spawning and the curriculum do not depend on the vocabulary, so they are the parent class's.

``scalar_oracle()`` is a context in which oracle/gen_golden.py builds this oracle for its traffic-junction cases
(scripts/gen_golden_tj_scalar.py writes the tj_scalar_* fixtures through it); ``make_env(args, tables)`` builds it from a
fixture's recorded args.
"""
import contextlib

import numpy as np

from oracle import gen_golden
from oracle import tj_env

OUTSIDE, ROAD, CAR, VOCAB = 0, 1, 2, 2


class TrafficJunctionScalarOracle(tj_env.TrafficJunctionOracle):
    def __init__(self, nagents, dim, vision, difficulty, tables, *a, **k):
        super(TrafficJunctionScalarOracle, self).__init__(nagents, dim, vision, difficulty, tables, *a, **k)
        self.BASE = None
        self.OUTSIDE, self.CAR, self.vocab_size = OUTSIDE, CAR, VOCAB
        self.obs_dim = 4 + self.W * self.W * VOCAB
        self.pad = np.pad(self.grid, self.vision, "constant", constant_values=OUTSIDE)

    def get_obs(self):
        """[N, 4 + W*W*2] float64 (flattened like env_wrappers.py:88-98)."""
        n, v, W = self.n, self.vision, self.W
        h, w = self.dims
        cnt = np.zeros((h + 2 * v, w + 2 * v), dtype=np.int64)
        for r, c in self.car_loc:                                 # every slot, dead ones sit at (0,0)
            cnt[r + v, c + v] += 1
        out = np.zeros((n, self.obs_dim), dtype=np.float64)
        for i in range(n):
            if not self.alive[i]:                                 # :352-356
                continue
            r, c = self.car_loc[i]
            win = np.zeros((W, W, VOCAB), dtype=np.float64)
            win[:, :, 0] = self.pad[r:r + W, c:c + W] == ROAD
            win[:, :, 1] = cnt[r:r + W, c:c + W]
            out[i, 0] = self.last_act[i] / (self.naction - 1)
            out[i, 1] = self.route_id[i] / (self.npath - 1)
            out[i, 2:4] = np.array([r, c]) / (h - 1, w - 1)         # float64 p_norm (:344)
            out[i, 4:] = win.reshape(-1)
        return out


def make_env(args, tables):
    return TrafficJunctionScalarOracle(args.nagents, args.dim, args.vision, args.difficulty, tables, args.add_rate_min,
                                       args.add_rate_max, args.curr_start, args.curr_end)


@contextlib.contextmanager
def scalar_oracle():
    """oracle.gen_golden's traffic-junction cases run the scalar-vocabulary oracle."""
    saved = gen_golden.make_oracle_env

    def make(args, tables=None):
        if args.env_name == "traffic_junction" and getattr(args, "vocab_type", "bool") == "scalar":
            return make_env(args, tables)
        return saved(args, tables)
    gen_golden.make_oracle_env = make
    try:
        yield
    finally:
        gen_golden.make_oracle_env = saved
