"""Batched traffic-junction environment on one GPU.

Same surface as the reference ``ic3net_envs/traffic_junction_env.py:TrafficJunctionEnv``
(``init_args`` :60-77, ``multi_agent_init`` :80-158, ``reset(epoch)`` :160-204, ``step``
:206-252, ``reward_terminal`` :611-612, ``curriculum`` :620-626, ``stat``), with
``args.nenvs`` independent junctions per instance advanced by csrc/tj_env.cu.  The
static tables (road-id grid, routes) are built once on the host
(ic3net_b200/traffic_helper.py) and uploaded.  obs is ``[B, N, 2 + W*W*V]`` float32
(already in the flattened order of env_wrappers.py:88-98); with ``vocab_type='scalar'``
(:139-148,331-332,344) it is ``[B, N, 4 + W*W*2]``: last action, route id, the car's
normalised position, then (is_road, car count) per window cell.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib, spaces, traffic_helper


class TrafficJunctionEnv(object):
    def __init__(self):
        self.__version__ = "0.0.1"
        self.OUTSIDE_CLASS = 0
        self.ROAD_CLASS = 1
        self.CAR_CLASS = 2
        self.TIMESTEP_PENALTY = -0.01
        self.CRASH_PENALTY = -10
        self.episode_over = False
        self.strict = True
        self.obs_version = 0    # bumped by every step / reset: validity of LazyObs handles (lazy_obs.py)
        self.obs_api = 'dense'  # 'handle': reset / step return a LazyObs instead of the dense tensor (args.obs_api)

    def init_args(self, parser):
        env = parser.add_argument_group('Traffic Junction task')
        env.add_argument('--dim', type=int, default=5, help="Dimension of box (i.e length of road) ")
        env.add_argument('--vision', type=int, default=1, help="Vision of car")
        env.add_argument('--add_rate_min', type=float, default=0.05,
                         help="rate at which to add car (till curr. start)")
        env.add_argument('--add_rate_max', type=float, default=0.2, help=" max rate at which to add car")
        env.add_argument('--curr_start', type=float, default=0,
                         help="start making harder after this many epochs [0]")
        env.add_argument('--curr_end', type=float, default=0, help="when to make the game hardest [0]")
        env.add_argument('--difficulty', type=str, default='easy', help="Difficulty level, easy|medium|hard")
        env.add_argument('--vocab_type', type=str, default='bool',
                         help="Type of location vector to use, bool|scalar")

    def multi_agent_init(self, args):
        _lib.require_cuda()
        self.obs_api = getattr(args, 'obs_api', 'dense')
        if self.obs_api not in ('dense', 'handle'):
            raise ValueError("obs_api must be 'dense' or 'handle'")
        for key in ('dim', 'vision', 'add_rate_min', 'add_rate_max', 'curr_start', 'curr_end', 'difficulty',
                    'vocab_type'):
            setattr(self, key, getattr(args, key))
        if self.vocab_type not in _lib.TJ_VOCAB:
            raise NotImplementedError("vocab_type must be 'bool' or 'scalar'")
        scalar = self.vocab_type == 'scalar'
        self.ncar = N = args.nagents
        t = traffic_helper.build_tables(self.difficulty, self.dim, self.vision, self.vocab_type)   # asserts of :93-100
        self.dims = list(t['dims'])
        self.exact_rate = self.add_rate = self.add_rate_min
        self.epoch_last_update = 0
        self.naction = 2
        self.action_space = spaces.Discrete(self.naction)
        self.npath = t['npath']
        if not scalar:
            self.BASE = t['BASE']              # the scalar vocabulary has none (:129-141)
        self.OUTSIDE_CLASS, self.CAR_CLASS, self.vocab_size = t['OUTSIDE'], t['CAR'], t['vocab']
        W = 2 * self.vision + 1
        # scalar: the position member is MultiDiscrete of the dims as given (:147), before easy's +1 -- only its
        # shape (2,) reaches observation_dim
        pos = [spaces.MultiDiscrete((self.dim, self.dim))] if scalar else []
        self.observation_space = spaces.Tuple([spaces.Discrete(self.naction), spaces.Discrete(self.npath)] + pos +
                                              [spaces.MultiBinary((W, W, self.vocab_size))])
        self.grid = t['grid']
        self.routes = t['routes']
        self.tables = t

        self.nenvs = B = int(getattr(args, 'nenvs', 1))
        self.device = dev = torch.device('cuda', torch.cuda.current_device())
        self.d_grid = torch.as_tensor(t['grid'].astype(np.int32)).to(dev).contiguous()
        self.d_route_len = torch.as_tensor(t['route_len']).to(dev).contiguous()
        self.d_route_cells = torch.as_tensor(t['route_cells']).to(dev).contiguous()
        self.cfg = _lib.TJCfg(B=B, N=N, vision=self.vision, h=self.dims[0], w=self.dims[1], G=t['G'], P=t['P'],
                              Lmax=t['Lmax'], outside_cls=self.OUTSIDE_CLASS, car_cls=self.CAR_CLASS,
                              vocab=self.vocab_size, npath=self.npath, spawn_thr=self._spawn_thr(),
                              vocab_type=_lib.TJ_VOCAB[self.vocab_type],
                              env_id0=int(getattr(args, 'env_id0', 0)),
                              seed=int(getattr(args, 'seed', 0)) & 0xFFFFFFFFFFFFFFFF,
                              grid=self.d_grid.data_ptr(), route_len=self.d_route_len.data_ptr(),
                              route_cells=self.d_route_cells.data_ptr())
        self.car_loc = torch.zeros(B, N, 2, dtype=torch.int32, device=dev)
        self.alive_mask = torch.zeros(B, N, dtype=torch.uint8, device=dev)
        self.wait = torch.zeros(B, N, dtype=torch.int32, device=dev)
        self.route_id = torch.full((B, N), -1, dtype=torch.int32, device=dev)
        self.car_route_loc = torch.full((B, N), -1, dtype=torch.int32, device=dev)
        self.car_last_act = torch.zeros(B, N, dtype=torch.uint8, device=dev)
        self.is_completed = torch.zeros(B, N, dtype=torch.uint8, device=dev)
        self.cars_in_sys = torch.zeros(B, dtype=torch.int32, device=dev)
        self.has_failed = torch.zeros(B, dtype=torch.uint8, device=dev)
        self.tick = torch.zeros(B, dtype=torch.int32, device=dev)
        self.err = torch.zeros(1, dtype=torch.int32, device=dev)
        self.state = _lib.TJState(loc=self.car_loc.data_ptr(), alive=self.alive_mask.data_ptr(),
                                  wait=self.wait.data_ptr(), route_id=self.route_id.data_ptr(),
                                  route_pos=self.car_route_loc.data_ptr(), last_act=self.car_last_act.data_ptr(),
                                  completed=self.is_completed.data_ptr(), cars_in_sys=self.cars_in_sys.data_ptr(),
                                  has_failed=self.has_failed.data_ptr(), tick=self.tick.data_ptr())
        self.obs_dim = (4 if scalar else 2) + W * W * self.vocab_size
        # encoder layout hint: two scalars, then cells of V entries whose last one (CAR) is a count; the scalar
        # vocabulary takes none (one plain sum: no per-position table, no fused index encoder, no BPTT kernels)
        self.obs_layout = (2, self.vocab_size, 1) if not scalar and self.CAR_CLASS == self.vocab_size - 1 else (0, 0, 0)
        self.obs_positions = self.dims[0] * self.dims[1]
        self.obs_shape = (B, N, self.obs_dim)
        self.stat = dict()
        return


    def chunk_view(self, k0, k1):
        """(cfg, state) of the env slots [k0, k1): the same device memory, for kernels run on a slice of the batch."""
        cfg = _lib.TJCfg.from_buffer_copy(self.cfg)
        cfg.B, cfg.env_id0 = k1 - k0, self.cfg.env_id0 + k0
        sl = lambda t: t[k0:k1].data_ptr()
        st = _lib.TJState(loc=sl(self.car_loc), alive=sl(self.alive_mask), wait=sl(self.wait), route_id=sl(self.route_id),
                          route_pos=sl(self.car_route_loc), last_act=sl(self.car_last_act),
                          completed=sl(self.is_completed), cars_in_sys=sl(self.cars_in_sys),
                          has_failed=sl(self.has_failed), tick=sl(self.tick))
        return cfg, st
    def _spawn_thr(self):
        # np.random.uniform() <= add_rate (:375) on 24-bit uniforms u = k * 2**-24
        return min(max(int(math.floor(self.add_rate * (2.0 ** 24))), 0), 0xFFFFFFFF) if self.add_rate >= 0 else 0

    def _new_obs(self):
        return torch.empty(self.obs_shape, dtype=torch.float32, device=self.device)

    _STATE = ('car_loc', 'alive_mask', 'wait', 'route_id', 'car_route_loc', 'car_last_act', 'is_completed', 'cars_in_sys', 'has_failed', 'tick')

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

    def reset(self, epoch=None, mask=None, want_obs=True):
        self.episode_over = False
        self.stat = dict()
        epoch_range = (self.curr_end - self.curr_start)
        add_rate_range = (self.add_rate_max - self.add_rate_min)
        if epoch is not None and epoch_range > 0 and add_rate_range > 0 and epoch > self.epoch_last_update:
            self.curriculum(epoch)
            self.epoch_last_update = epoch
        self.obs_version += 1
        lazy = want_obs and self.obs_api == 'handle'
        obs = self._new_obs() if (want_obs and not lazy) else None
        m = None if mask is None else torch.as_tensor(mask).to(self.device, torch.uint8).contiguous()
        _lib.check(_lib.load().ic3_tj_reset(C.byref(self.cfg), C.byref(self.state), _lib.ptr(m), _lib.ptr(obs),
                                            _lib.stream()))
        return self._obs_handle() if lazy else obs

    def curriculum(self, epoch):
        step_size = 0.01
        step = (self.add_rate_max - self.add_rate_min) / (self.curr_end - self.curr_start)
        if self.curr_start <= epoch < self.curr_end:
            self.exact_rate = self.exact_rate + step
            self.add_rate = step_size * (self.exact_rate // step_size)
            self.cfg.spawn_thr = self._spawn_thr()

    def curriculum_until(self, epoch):
        """add_rate as training reaches it at `epoch`: the curriculum replayed from add_rate_min through reset(1) ..
        reset(epoch) (the final epoch gives the target add_rate)."""
        self.exact_rate = self.add_rate = self.add_rate_min
        self.epoch_last_update = 0
        self.cfg.spawn_thr = self._spawn_thr()
        if self.curr_end - self.curr_start > 0 and self.add_rate_max - self.add_rate_min > 0:
            for ep in range(1, epoch + 1):
                self.curriculum(ep)
                self.epoch_last_update = ep

    def set_add_rate(self, other):
        """Take the curriculum state (add_rate and its progress) of another env of the same configuration."""
        self.exact_rate, self.add_rate, self.epoch_last_update = other.exact_rate, other.add_rate, other.epoch_last_update
        self.cfg.spawn_thr = self._spawn_thr()

    def _get_obs(self):
        obs = self._new_obs()
        _lib.check(_lib.load().ic3_tj_obs(C.byref(self.cfg), C.byref(self.state), obs.data_ptr(), _lib.stream()))
        return obs

    def check_errors(self):
        flags = int(self.err.item())
        if flags:
            self.err.zero_()
        if flags & _lib.ERR_ROUTE_OVERRUN:
            raise RuntimeError("Out of boud car path")
        if flags & _lib.ERR_BAD_ACTION:
            raise AssertionError("Actions should be in the range [0,naction).")

    def step(self, action, draws=None, obs_out=None):
        a = action if torch.is_tensor(action) else torch.as_tensor(np.asarray(action))
        assert a.numel() == self.nenvs * self.ncar, "Action for each agent should be provided."
        act = a.to(self.device, torch.int32, non_blocking=True).reshape(self.nenvs, self.ncar).contiguous()
        d = None
        if draws is not None:      # explicit 24-bit draws [B, G, 3] instead of the Philox spawn stream
            d = torch.as_tensor(np.asarray(draws, dtype=np.int64)).to(self.device, torch.int32).contiguous()
            assert d.numel() == self.nenvs * self.cfg.G * 3
        reward = torch.empty(self.nenvs, self.ncar, dtype=torch.float32, device=self.device)
        lazy = obs_out is None and self.obs_api == 'handle'
        obs = None if lazy else (self._new_obs() if obs_out is None else obs_out)
        self.obs_version += 1
        _lib.check(_lib.load().ic3_tj_step(C.byref(self.cfg), C.byref(self.state), act.data_ptr(), 1, _lib.ptr(d),
                                           reward.data_ptr(), _lib.ptr(obs), self.err.data_ptr(), None,
                                           _lib.stream()))
        if lazy:
            obs = self._obs_handle()
        if self.strict:
            self.check_errors()
        debug = {'car_loc': self.car_loc, 'alive_mask': self.alive_mask.clone(), 'wait': self.wait,
                 'cars_in_sys': self.cars_in_sys, 'is_completed': self.is_completed.clone()}
        done = torch.zeros(self.nenvs, dtype=torch.bool, device=self.device)   # never set by the reference (:252)
        return obs, reward, done, debug

    def reward_terminal(self):
        return torch.zeros(self.nenvs, self.ncar, dtype=torch.float32, device=self.device)

    def get_stat(self):
        self.stat['success'] = int((1 - self.has_failed.int()).sum().item())
        self.stat['add_rate'] = self.add_rate * self.nenvs
        return self.stat

    def seed(self):
        return

    def render(self, mode='human', close=False):
        raise NotImplementedError("curses rendering is not part of the accelerated path")

    def exit_render(self):
        raise NotImplementedError("curses rendering is not part of the accelerated path")
