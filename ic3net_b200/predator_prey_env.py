"""Batched predator-prey environment on one GPU.

Same surface as the reference ``ic3net_envs/predator_prey_env.py:PredatorPreyEnv``
(``init_args`` :55-70, ``multi_agent_init`` :72-110, ``reset`` :146-168, ``step``
:112-144, ``reward_terminal`` :292-293, ``stat``, ``observation_space``,
``action_space``, ``naction``, ``vocab_size``), but one instance holds
``args.nenvs`` independent environments whose state lives in HBM and is advanced
by the CUDA kernels in csrc/pp_env.cu.  Returned arrays are CUDA tensors with a
leading env dimension: obs ``[B, N, W, W, V]`` float32, reward ``[B, N]`` float32,
done ``[B]`` bool; info holds live views of the state like the reference does.  With
``--enemy_comm`` the prey is one more agent row (N + 1 rows of obs / reward / action).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib, spaces


class PredatorPreyEnv(object):
    def __init__(self):
        self.__version__ = "0.0.1"
        self.TIMESTEP_PENALTY = -0.05
        self.PREY_REWARD = 0
        self.POS_PREY_REWARD = 0.05
        self.episode_over = False
        self.strict = True      # raise "Episode is done" eagerly (one 4-byte host read per step)
        self.obs_version = 0    # bumped by every step / reset: validity of LazyObs handles (lazy_obs.py)
        self.obs_api = 'dense'  # 'handle': reset / step return a LazyObs instead of the dense tensor (args.obs_api)

    def init_args(self, parser):
        env = parser.add_argument_group('Prey Predator task')
        env.add_argument('--nenemies', type=int, default=1, help="Total number of preys in play")
        env.add_argument('--dim', type=int, default=5, help="Dimension of box")
        env.add_argument('--vision', type=int, default=2, help="Vision of predator")
        env.add_argument('--moving_prey', action="store_true", default=False,
                         help="Whether prey is fixed or moving")
        env.add_argument('--no_stay', action="store_true", default=False,
                         help="Whether predators have an action to stay in place")
        parser.add_argument('--mode', default='mixed', type=str,
                            help='cooperative|competitive|mixed (default: mixed)')
        env.add_argument('--enemy_comm', action="store_true", default=False,
                         help="Whether prey can communicate.")

    def multi_agent_init(self, args):
        _lib.require_cuda()
        self.obs_api = getattr(args, 'obs_api', 'dense')
        if self.obs_api not in ('dense', 'handle'):
            raise ValueError("obs_api must be 'dense' or 'handle'")
        for key in ('dim', 'vision', 'moving_prey', 'mode', 'enemy_comm'):
            setattr(self, key, getattr(args, key))
        self.nprey = args.nenemies
        self.npredator = args.nfriendly
        self.dims = (self.dim, self.dim)
        self.stay = not args.no_stay
        if args.moving_prey:
            raise NotImplementedError           # predator_prey_env.py:84-85
        if self.nprey != 1:
            raise NotImplementedError("nenemies != 1: the reference reward logic only works for one prey (:258)")
        if self.mode not in _lib.PP_MODES:       # :269
            raise RuntimeError("Incorrect mode, Available modes: [cooperative|competitive|mixed]")
        self.naction = 5 if self.stay else 4
        self.action_space = spaces.MultiDiscrete([self.naction])
        self.BASE = self.dim * self.dim
        self.OUTSIDE_CLASS, self.PREY_CLASS, self.PREDATOR_CLASS = self.BASE + 1, self.BASE + 2, self.BASE + 3
        self.vocab_size = self.BASE + 4
        W = 2 * self.vision + 1
        self.observation_space = spaces.Box(low=0, high=1, shape=(self.vocab_size, W, W), dtype=int)

        self.nenvs = B = int(getattr(args, 'nenvs', 1))
        N = self.npredator
        # --enemy_comm (:203-207, :255, :276-281): the prey is agent row N of obs / reward / action (action ignored)
        self.nagent_rows = NA = N + (1 if self.enemy_comm else 0)
        self.device = torch.device('cuda', torch.cuda.current_device())
        seed = int(getattr(args, 'seed', 0))
        self.cfg = _lib.PPCfg(B=B, N=N, dim=self.dim, vision=self.vision, mode=_lib.PP_MODES[self.mode],
                              naction=self.naction, env_id0=int(getattr(args, 'env_id0', 0)),
                              enemy_comm=int(bool(self.enemy_comm)), seed=seed & 0xFFFFFFFFFFFFFFFF)
        dev = self.device
        self.loc = torch.zeros(B, N + 1, 2, dtype=torch.int32, device=dev)
        self.reached_prey = torch.zeros(B, N, dtype=torch.uint8, device=dev)
        self.done = torch.zeros(B, dtype=torch.uint8, device=dev)
        self.success = torch.full((B,), -1, dtype=torch.int32, device=dev)
        self.episode = torch.zeros(B, dtype=torch.int32, device=dev)
        self.tick = torch.zeros(B, dtype=torch.int32, device=dev)
        self.err = torch.zeros(1, dtype=torch.int32, device=dev)
        self.state = _lib.PPState(loc=self.loc.data_ptr(), reached=self.reached_prey.data_ptr(),
                                  done=self.done.data_ptr(), success=self.success.data_ptr(),
                                  episode=self.episode.data_ptr(), tick=self.tick.data_ptr())
        self.obs_shape = (B, NA, W, W, self.vocab_size)
        self.obs_dim = W * W * self.vocab_size
        # encoder layout hint (ic3_policy_cfg.obs_off / obs_vocab / obs_ncount): cells of V entries, last two = counts
        self.obs_layout = (0, self.vocab_size, 2)
        self.obs_positions = self.dim * self.dim
        self.stat = dict()
        return

    def chunk_view(self, k0, k1):
        """(cfg, state) of the env slots [k0, k1): the same device memory, for kernels run on a slice of the batch."""
        cfg = _lib.PPCfg.from_buffer_copy(self.cfg)
        cfg.B, cfg.env_id0 = k1 - k0, self.cfg.env_id0 + k0
        st = _lib.PPState(loc=self.loc[k0:k1].data_ptr(), reached=self.reached_prey[k0:k1].data_ptr(),
                          done=self.done[k0:k1].data_ptr(), success=self.success[k0:k1].data_ptr(),
                          episode=self.episode[k0:k1].data_ptr(), tick=self.tick[k0:k1].data_ptr())
        return cfg, st

    # views with the reference's names (predator_prey_env.py:158-159)
    @property
    def predator_loc(self):
        return self.loc[:, :self.npredator]

    @property
    def prey_loc(self):
        return self.loc[:, self.npredator:]

    def _new_obs(self):
        return torch.empty(self.obs_shape, dtype=torch.float32, device=self.device)

    _STATE = ('loc', 'reached_prey', 'done', 'success', 'episode', 'tick')

    def snapshot(self):
        """Copy of the whole device state of the batch (positions, flags, RNG counters): restore() rewinds to it."""
        return [getattr(self, k).clone() for k in self._STATE]

    def restore(self, snap):
        for k, v in zip(self._STATE, snap):
            getattr(self, k).copy_(v)
        self.obs_version += 1

    def _obs_handle(self):
        from .lazy_obs import LazyObs
        return LazyObs(self)

    def set_state(self, predator_loc, prey_loc):
        """Inject spawn positions (parity tests / replays) instead of sampling them."""
        loc = torch.as_tensor(np.concatenate([np.asarray(predator_loc).reshape(self.nenvs, self.npredator, 2),
                                              np.asarray(prey_loc).reshape(self.nenvs, 1, 2)], 1))
        self.loc.copy_(loc.to(self.device, torch.int32))
        self.reached_prey.zero_()
        self.done.zero_()
        self.success.fill_(-1)
        self.episode_over = False
        return self._get_obs()

    def reset(self, mask=None, want_obs=True):
        self.episode_over = False
        self.obs_version += 1
        lazy = want_obs and self.obs_api == 'handle'
        obs = self._new_obs() if (want_obs and not lazy) else None
        m = None if mask is None else torch.as_tensor(mask).to(self.device, torch.uint8).contiguous()
        _lib.check(_lib.load().ic3_pp_reset(C.byref(self.cfg), C.byref(self.state), _lib.ptr(m), _lib.ptr(obs),
                                            _lib.stream()))
        self.stat = dict()
        return self._obs_handle() if lazy else obs

    def _get_obs(self):
        obs = self._new_obs()
        _lib.check(_lib.load().ic3_pp_obs(C.byref(self.cfg), C.byref(self.state), obs.data_ptr(), _lib.stream()))
        return obs

    def _as_action(self, action):
        a = action if torch.is_tensor(action) else torch.as_tensor(np.asarray(action))
        a = a.to(self.device, torch.int32, non_blocking=True).reshape(self.nenvs, self.nagent_rows).contiguous()
        return a

    def check_errors(self):
        flags = int(self.err.item())
        if flags:
            self.err.zero_()
        if flags & _lib.ERR_EPISODE_DONE:
            raise RuntimeError("Episode is done")
        if flags & _lib.ERR_BAD_ACTION:
            raise AssertionError("Actions should be in the range [0,naction).")

    def step(self, action, obs_out=None):
        act = self._as_action(action)
        reward = torch.empty(self.nenvs, self.nagent_rows, dtype=torch.float32, device=self.device)
        lazy = obs_out is None and self.obs_api == 'handle'
        obs = None if lazy else (self._new_obs() if obs_out is None else obs_out)
        self.obs_version += 1
        _lib.check(_lib.load().ic3_pp_step(C.byref(self.cfg), C.byref(self.state), act.data_ptr(), 1,
                                           reward.data_ptr(), _lib.ptr(obs), self.err.data_ptr(), None,
                                           _lib.stream()))
        if lazy:
            obs = self._obs_handle()
        if self.strict:
            self.check_errors()
        done = self.done.bool()
        self.episode_over = done
        debug = {'predator_locs': self.predator_loc, 'prey_locs': self.prey_loc}
        return obs, reward, done, debug

    def reward_terminal(self):
        # the reference re-runs _get_reward here (side effects only, idempotent on an
        # unchanged state) and returns zeros (:292-293)
        return torch.zeros(self.nenvs, self.nagent_rows, dtype=torch.float32, device=self.device)

    def get_stat(self):
        """stat['success'] summed over the envs of the batch (host read)."""
        if self.mode != 'competitive':
            self.stat['success'] = int(self.success.clamp(min=0).sum().item())
        return self.stat

    def seed(self):
        return

    def render(self, mode='human', close=False):
        raise NotImplementedError("curses rendering is not part of the accelerated path")

    def exit_render(self):
        raise NotImplementedError("curses rendering is not part of the accelerated path")
